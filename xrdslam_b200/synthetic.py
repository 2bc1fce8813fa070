"""Synthetic 640x480 RGB-D sequence (SURVEY.md section 8d): an analytic room box
with two inner boxes, depth by exact ray/plane intersection, smooth procedural
colour, camera on a circle looking at the room centre (OpenGL c2w convention,
as the reference's loaders produce, slam/common/datasets.py:154-163)."""
from __future__ import annotations

import numpy as np

from .camera import Camera

ROOM = np.array([[-2.9, 2.9], [-3.9, 2.4], [-1.9, 2.4]])
BOXES = [np.array([[0.8, 1.8], [-0.2, 0.9], [-1.9, -0.7]]),
         np.array([[-2.0, -1.1], [-2.5, -1.3], [-1.9, 0.1]])]
CENTRE = np.array([0.0, -0.75, 0.25])


def make_camera(width=640, height=480):
    f = 320.0 * width / 640.0
    return Camera(f, f, (width - 1) / 2.0, (height - 1) / 2.0, width, height)


def look_at(eye, target, up=np.array([0.0, 0.0, 1.0])):
    f = target - eye
    f = f / np.linalg.norm(f)
    x = np.cross(f, up)
    x = x / np.linalg.norm(x)
    y = np.cross(x, f)
    c2w = np.eye(4)
    c2w[:3, 0], c2w[:3, 1], c2w[:3, 2], c2w[:3, 3] = x, y, -f, eye
    return c2w.astype(np.float32)


def trajectory(n_frames, radius=0.8, offset=(0.0, 0.0, 0.0)):
    poses = []
    for k in range(n_frames):
        a = 2 * np.pi * k / max(n_frames, 1) * 0.25  # quarter turn over the run
        eye = CENTRE + np.array([radius * np.cos(a), radius * np.sin(a), 0.1])
        tgt = CENTRE + np.array([-1.5 * np.cos(a + 0.6), -1.5 * np.sin(a + 0.6), -0.3])
        c2w = look_at(eye, tgt)
        c2w[:3, 3] += np.asarray(offset, dtype=np.float32)
        poses.append(c2w)
    return poses


def _slab(o, d, box):
    with np.errstate(divide='ignore', invalid='ignore'):
        t0 = (box[:, 0] - o) / d
        t1 = (box[:, 1] - o) / d
    tn = np.minimum(t0, t1).max(-1)
    tf = np.maximum(t0, t1).min(-1)
    return tn, tf


def render_frame(camera: Camera, c2w, offset=(0.0, 0.0, 0.0), invalid_frac=0.02,
                 seed=0):
    """-> rgb [H,W,3] f32 in [0,1], depth [H,W] f32 (z-depth, 0 = invalid)."""
    H, W = camera.height, camera.width
    j, i = np.meshgrid(np.arange(H, dtype=np.float64),
                       np.arange(W, dtype=np.float64), indexing='ij')
    dirs = np.stack([(i - camera.cx) / camera.fx, -(j - camera.cy) / camera.fy,
                     -np.ones_like(i)], -1)
    c2w = np.asarray(c2w, dtype=np.float64)
    off = np.asarray(offset, dtype=np.float64)
    d = dirs @ c2w[:3, :3].T
    o = c2w[:3, 3] - off
    _, t = _slab(o, d, ROOM)  # camera is inside: exit distance
    for b in BOXES:
        tn, tf = _slab(o, d, b)
        hit = (tn < tf) & (tn > 0)
        t = np.where(hit & (tn < t), tn, t)
    p = o + d * t[..., None]
    rgb = 0.5 + 0.5 * np.sin(p @ np.array([[2.1, 0.7, 1.3], [0.9, 2.3, 0.5],
                                           [1.1, 0.6, 2.7]]) + np.array([0.3, 1.1, 2.0]))
    depth = t.copy()  # |dir_z| == 1 -> ray parameter == z-depth
    rng = np.random.default_rng(seed)
    depth[rng.random((H, W)) < invalid_frac] = 0.0
    return rgb.astype(np.float32), depth.astype(np.float32)


def make_sequence(n_frames, width=640, height=480, offset=(0.0, 0.0, 0.0)):
    cam = make_camera(width, height)
    poses = trajectory(n_frames, offset=offset)
    frames = [render_frame(cam, p, offset=offset, seed=k)
              for k, p in enumerate(poses)]
    return cam, poses, frames


def _grid_rect(origin, u, v, nu, nv):
    """A rectangle origin + [0,1]u + [0,1]v as an (nu x nv)-cell triangle grid."""
    a, b = np.meshgrid(np.linspace(0.0, 1.0, nu + 1), np.linspace(0.0, 1.0, nv + 1), indexing='ij')
    verts = origin + a.reshape(-1, 1) * u + b.reshape(-1, 1) * v
    idx = np.arange((nu + 1) * (nv + 1)).reshape(nu + 1, nv + 1)
    q = np.stack([idx[:-1, :-1], idx[1:, :-1], idx[1:, 1:], idx[:-1, 1:]], -1).reshape(-1, 4)
    faces = np.concatenate([q[:, [0, 1, 2]], q[:, [0, 2, 3]]])
    return verts, faces


def room_mesh(spacing=0.1):
    """The analytic scene (ROOM's six walls and the BOXES' faces that do not lie on a wall) as a
    triangle mesh with vertices about `spacing` apart: -> (verts f32 [V,3], faces i32 [F,3]).
    The ground truth the reconstruction tests score against."""
    verts, faces, base = [], [], 0

    def box_faces(box, skip_walls):
        for ax in range(3):
            u_ax, v_ax = [a for a in range(3) if a != ax]
            for side in range(2):
                if skip_walls and box[ax, side] in (ROOM[ax, 0], ROOM[ax, 1]):
                    continue
                o = box[:, 0].astype(np.float64).copy()
                o[ax] = box[ax, side]
                u = np.zeros(3)
                v = np.zeros(3)
                u[u_ax] = box[u_ax, 1] - box[u_ax, 0]
                v[v_ax] = box[v_ax, 1] - box[v_ax, 0]
                yield o, u, v

    rects = list(box_faces(ROOM, False))
    for b in BOXES:
        rects += list(box_faces(b, True))
    for o, u, v in rects:
        nu = max(1, int(round(np.linalg.norm(u) / spacing)))
        nv = max(1, int(round(np.linalg.norm(v) / spacing)))
        vv, ff = _grid_rect(o, u, v, nu, nv)
        verts.append(vv)
        faces.append(ff + base)
        base += len(vv)
    return np.concatenate(verts).astype(np.float32), np.concatenate(faces).astype(np.int32)
