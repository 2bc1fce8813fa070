"""cull_mesh (slam/common/common.py:714-789, reference @ f0366f20) restated twice.

(a) ``visible`` / ``compact``: numpy float32 with csrc/cull.cu's exact operation order (the
    semantics in include/xrdslam_b200.h).  It is the CUDA kernels' oracle, bit for bit.
(b) ``reference_seen``: the reference's per-frame loop in device-agnostic torch (torch.inverse,
    the broadcast matmuls, F.grid_sample, the mask), OR-ed into a mask on the device instead of
    ANDed into a host array.  On the CPU it is bit-identical to the reference's own function
    (tests/test_cull_cpu.py); on the GPU it is the reference's arithmetic on the real device.

(a) and (b) need not agree bit for bit: torch's matmul and grid_sample may round differently
(summation order, vectorised unnormalise, FMA).  ``borderline`` is the rule the tests use for
a disagreement: some frame's decision flips when recomputed in float64 with u, v perturbed by
+-1e-3 px and depth by +-1e-5 m.
"""
from __future__ import annotations

import numpy as np

f32 = np.float32


def _intr(cam):
    return int(cam.height), int(cam.width), f32(cam.fx), f32(cam.fy), f32(cam.cx), f32(cam.cy)


def _sample_depth(D, u, v, H, W):
    """grid_sample(bilinear, zeros, align_corners=True) at 2 * (u / W, v / H) - 1, float32 in
    csrc/cull.cu's order (corners nw, ne, sw, se added to 0 when inside the image)."""
    gx = f32(2) * (u / f32(W)) - f32(1)
    gy = f32(2) * (v / f32(H)) - f32(1)
    ix = ((gx + f32(1)) / f32(2)) * f32(W - 1)
    iy = ((gy + f32(1)) / f32(2)) * f32(H - 1)
    x0, y0 = np.floor(ix), np.floor(iy)
    x1, y1 = x0 + f32(1), y0 + f32(1)
    w = [(x1 - ix) * (y1 - iy), (ix - x0) * (y1 - iy), (x1 - ix) * (iy - y0), (ix - x0) * (iy - y0)]
    c0, r0 = x0.astype(np.int64), y0.astype(np.int64)
    d = np.zeros(u.shape, f32)
    for (r, c), wk in zip(((r0, c0), (r0, c0 + 1), (r0 + 1, c0), (r0 + 1, c0 + 1)), w):
        m = (r >= 0) & (r < H) & (c >= 0) & (c < W)
        d[m] = d[m] + D[r[m], c[m]] * wk[m]
    return d


def visible(verts, w2c, depth, cam, truncation=0.06, eval_rec=False, seen=None):
    """Vertices f32 [V,3], w2c f32 [F,3,4] (or [F,4,4]), depth f32 [F,H,W] -> seen bool [V]
    (OR-ed into a copy of `seen` if given): xrd_cull_visible."""
    p = np.asarray(verts, f32).reshape(-1, 3)
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    H, W, fx, fy, cx, cy = _intr(cam)
    trunc = f32(truncation)
    seen = np.zeros(p.shape[0], bool) if seen is None else np.asarray(seen, bool).copy()
    for f in range(len(w2c)):
        T = np.asarray(w2c[f], f32)
        row = lambda r: ((T[r, 0] * x + T[r, 1] * y) + T[r, 2] * z) + T[r, 3]
        with np.errstate(all='ignore'):
            xc, yc, zc = -row(0), row(1), row(2)
            up = fx * xc + cx * zc
            vp = fy * yc + cy * zc
            zz = zc + f32(1e-5)
            u, v = up / zz, vp / zz
            ok = (f32(0) <= -zz) & (u < f32(W)) & (u > f32(0)) & (v < f32(H)) & (v > f32(0))
            if eval_rec:
                i = np.nonzero(ok & ~seen)[0]
                d = _sample_depth(np.asarray(depth[f], f32), u[i], v[i], H, W)
                ok[:] = False
                ok[i] = (d + trunc) >= -zz[i]
        seen |= ok
    return seen


def compact(seen, verts, faces, colors=None):
    """xrd_cull_count / xrd_cull_emit: keep the faces with a seen vertex and the vertices they
    reference, both in order; faces remapped; colours follow.  -> (verts, faces i32, colours)."""
    seen = np.asarray(seen, bool)
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    keep = seen[faces].any(1) if faces.shape[0] else np.zeros(0, bool)
    ref = np.zeros(seen.shape[0], bool)
    ref[faces[keep].reshape(-1)] = True
    new_id = np.cumsum(ref) - 1
    out_c = None if colors is None else np.asarray(colors)[ref]
    return (np.asarray(verts, f32).reshape(-1, 3)[ref], new_id[faces[keep]].astype(np.int32),
            out_c)


def reference_seen(dataset, vertices, estimate_c2w_list=None, eval_rec=False, truncation=0.06,
                   device='cpu'):
    """(b): the reference's visibility loop in torch on `device` -> seen bool [V] (the reference's
    ~whole_mask) on that device."""
    import torch
    import torch.nn.functional as F
    n_imgs = len(estimate_c2w_list) if estimate_c2w_list is not None else len(dataset)
    cam = dataset.get_camera()
    H, W = cam.height, cam.width
    pts = torch.as_tensor(vertices).to(device)
    homo = torch.cat([pts, torch.ones_like(pts[:, :1])], 1).reshape(-1, 4, 1).float()
    K = torch.from_numpy(np.array([[cam.fx, 0.0, cam.cx], [0.0, cam.fy, cam.cy],
                                   [0.0, 0.0, 1.0]])).to(device).float()
    seen = torch.zeros(pts.shape[0], dtype=torch.bool, device=device)
    for i in range(n_imgs):
        _, _, depth, c2w = dataset[i]
        if estimate_c2w_list is not None:
            c2w = estimate_c2w_list[i]
        depth, c2w = torch.as_tensor(depth).to(device), torch.as_tensor(c2w).to(device)
        xyz = (torch.inverse(c2w) @ homo)[:, :3]
        xyz[:, 0] *= -1
        uvz = K @ xyz
        z = uvz[:, -1:] + 1e-5
        uv = (uvz[:, :2] / z).squeeze(-1)
        g = uv[None, None].clone()
        g[..., 0] = g[..., 0] / W
        g[..., 1] = g[..., 1] / H
        g = 2 * g - 1
        d = F.grid_sample(depth[None, None], g, padding_mode='zeros',
                          align_corners=True).reshape(-1)
        zn = -z[:, 0, 0]
        vis = (0 <= zn) & (uv[:, 0] < W) & (uv[:, 0] > 0) & (uv[:, 1] < H) & (uv[:, 1] > 0)
        if eval_rec:
            vis = vis & (d + truncation >= zn)
        seen |= vis
    return seen


def _sample_depth64(D, u, v, H, W):
    ix, iy = u / W * (W - 1), v / H * (H - 1)
    x0, y0 = np.floor(ix), np.floor(iy)
    d = np.zeros(u.shape)
    for dr, dc, w in ((0, 0, (x0 + 1 - ix) * (y0 + 1 - iy)), (0, 1, (ix - x0) * (y0 + 1 - iy)),
                      (1, 0, (x0 + 1 - ix) * (iy - y0)), (1, 1, (ix - x0) * (iy - y0))):
        r, c = y0.astype(np.int64) + dr, x0.astype(np.int64) + dc
        m = (r >= 0) & (r < H) & (c >= 0) & (c < W)
        d[m] += D[r[m], c[m]] * w[m]
    return d


def borderline(verts, w2c, depth, cam, truncation=0.06, eval_rec=False, du=1e-3, dd=1e-5):
    """bool [V]: for some frame, the float64 decision is not the same for every combination of
    u, v shifted by -du, 0, +du px and depth (and -z) by -dd, 0, +dd m."""
    p = np.asarray(verts, np.float64).reshape(-1, 3)
    H, W = int(cam.height), int(cam.width)
    fx, fy, cx, cy = (float(f32(a)) for a in (cam.fx, cam.fy, cam.cx, cam.cy))
    out = np.zeros(p.shape[0], bool)
    if p.shape[0] == 0:
        return out
    steps = (-1.0, 0.0, 1.0)
    for f in range(len(w2c)):
        T = np.asarray(w2c[f], np.float64)[:3]
        c = p @ T[:, :3].T + T[:, 3]
        with np.errstate(all='ignore'):
            z = c[:, 2] + float(f32(1e-5))
            u = (-fx * c[:, 0] + cx * c[:, 2]) / z
            v = (fy * c[:, 1] + cy * c[:, 2]) / z
            dec = []
            for su in steps:
                for sv in steps:
                    uu, vv = u + su * du, v + sv * du
                    ins = (uu > 0) & (uu < W) & (vv > 0) & (vv < H)
                    d = np.zeros(p.shape[0])
                    if eval_rec:
                        d[ins] = _sample_depth64(np.asarray(depth[f], np.float64), uu[ins], vv[ins],
                                                 H, W)
                    for sd in steps:
                        ok = ins & (0 <= -z + sd * dd)
                        if eval_rec:
                            ok &= d + sd * dd + float(f32(truncation)) >= -z
                        dec.append(ok)
        dec = np.stack(dec)
        out |= dec.any(0) != dec.all(0)
    return out
