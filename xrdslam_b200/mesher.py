"""Mesh extraction (host-side mirror of slam/common/mesher.py, reference @ f0366f20).

The reference evaluates the scene function on a resolution^3 lattice, copies every value to
the host and runs skimage's marching cubes there; the vertices then go back through the
colour function.  Here the lattice points are generated on the device in volume order (x
slowest), the queries fill a device volume, marching cubes runs in csrc/mesh.cu and only the
mesh itself (vertices, faces, uint8 colours) is copied to the host.  skimage / trimesh /
open3d are not needed: ``TriMesh`` holds the arrays and writes the binary PLY the tracker's
``final_mesh.ply`` is (io_formats.write_ply).
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import Type

import numpy as np
import torch

from . import _cabi
from ._cabi import XrdMeshAffine, ptr
from .base_model import InstantiateConfig


@dataclass
class MesherConfig(InstantiateConfig):
    """mesher.py:19-29 (field names and defaults kept)."""
    _target: Type = field(default_factory=lambda: Mesher)
    points_batch_size: int = 500000
    resolution: int = 130
    level_set: int = 0
    remove_small_geometry_threshold: float = 0.2
    clean_mesh_bound_scale: float = 1.02
    get_largest_components: bool = False


class TriMesh:
    """The parts of trimesh.Trimesh the tracker uses: host arrays and ``export``."""

    def __init__(self, vertices, faces, vertex_colors=None):
        self.vertices = vertices            # f32 [V,3]
        self.faces = faces                  # i32 [F,3]
        self.vertex_colors = vertex_colors  # u8 [V,3] or None

    def export(self, path):
        from .io_formats import write_ply
        return write_ply(path, self.vertices, self.faces, self.vertex_colors)


def marching_cubes(values, level, spacing, shift=(0.0, 0.0, 0.0), scale=(1.0, 1.0, 1.0),
                   origin=None):
    """csrc/mesh.cu on DEVICE values f32 [B,nx,ny,nz] -> DEVICE verts f32 [V,3], faces i32 [F,3].
    World coordinates ((p * spacing + shift) * scale) + origin[b] (fp32), origin [B,3] or None;
    semantics in include/xrdslam_b200.h.  One host read: the two totals."""
    _cabi.require_cuda(values.device, 'values')
    dev = values.device
    vals = values.detach().to(torch.float32).contiguous()
    B, nx, ny, nz = vals.shape
    ws, nb = _cabi.workspace(
        dev, 'mesh_mc', B, nx, ny, nz,
        error=f'marching cubes needs B >= 1 and nx, ny, nz >= 2, got {tuple(vals.shape)}')
    counts = torch.empty(2, dtype=torch.int32, device=dev)
    org = None if origin is None else origin.detach().to(dev, torch.float32).contiguous()
    if org is not None and tuple(org.shape) != (B, 3):
        raise ValueError('origin must be [B,3]')
    f3 = lambda a: (C.c_float * 3)(*[float(x) for x in a])
    aff = XrdMeshAffine(f3(spacing), f3(shift), f3(scale), ptr(org))
    with torch.cuda.device(dev):
        _cabi.launch_on(dev, 'xrd_mesh_mc_count', ptr(vals), B, nx, ny, nz, float(level),
                        ptr(counts), ptr(ws), nb)
        V, F = counts.tolist()
        verts = torch.empty(V, 3, dtype=torch.float32, device=dev)
        faces = torch.empty(F, 3, dtype=torch.int32, device=dev)
        _cabi.launch_on(dev, 'xrd_mesh_mc_emit', ptr(vals), B, nx, ny, nz, float(level),
                        C.byref(aff), ptr(verts), ptr(faces), ptr(ws), nb)
    return verts, faces


def colors_to_u8(c):
    """mesher.py:251-253: clip(0, 1) * 255 cast to uint8 (truncation), on the device."""
    return (c.clamp(0, 1) * 255).to(torch.uint8)


class Mesher():
    def __init__(self, config: MesherConfig, camera, bounding_box, marching_cubes_bound) -> None:
        self.config = config
        self.bounding_box = bounding_box
        self.marching_cubes_bound = marching_cubes_bound
        self.camera = camera
        self.scale = 1.0

    def get_grid_uniform(self, resolution):
        """mesher.py:40-67: the lattice axes (np.linspace, float64).  The reference also builds
        the [resolution^3, 3] point tensor here; ``grid_points`` makes it on the device, chunk
        by chunk, instead."""
        bound = self.marching_cubes_bound
        padding = 0.0
        x = np.linspace(float(bound[0][0]) - padding, float(bound[0][1]) + padding, resolution)
        y = np.linspace(float(bound[1][0]) - padding, float(bound[1][1]) + padding, resolution)
        z = np.linspace(float(bound[2][0]) - padding, float(bound[2][1]) + padding, resolution)
        return {'xyz': [x, y, z]}

    @staticmethod
    def grid_points(xyz, start, count, device):
        """Lattice points f32 [count,3] of flat volume indices start .. start+count-1 (x slowest,
        the marching-cubes layout), generated on `device`.  Coordinates are the float64 axes
        rounded to float32, as torch.tensor(..., dtype=torch.float) does in the reference."""
        ax = [torch.as_tensor(a, dtype=torch.float64).to(device=device, dtype=torch.float32)
              for a in xyz]
        ny, nz = len(xyz[1]), len(xyz[2])
        idx = torch.arange(start, start + count, device=device)
        return torch.stack([ax[0][idx // (ny * nz)], ax[1][(idx // nz) % ny], ax[2][idx % nz]], -1)

    def eval_points(self, p, query_fn, boundingbox, device='cuda:0'):
        """mesher.py:147-177: query_fn per points_batch_size chunk; 100 outside the bound (the
        float32 points compare with the float64 0-dim bounds in float32, as in the reference)."""
        p_split = torch.split(p, self.config.points_batch_size)
        bound = boundingbox
        rets = []
        for pi in p_split:
            mask_x = (pi[:, 0] < bound[0][1]) & (pi[:, 0] > bound[0][0])
            mask_y = (pi[:, 1] < bound[1][1]) & (pi[:, 1] > bound[1][0])
            mask_z = (pi[:, 2] < bound[2][1]) & (pi[:, 2] > bound[2][0])
            mask = mask_x & mask_y & mask_z
            ret = query_fn(pi)
            ret[~mask, :] = 100
            rets.append(ret)
        return torch.cat(rets, dim=0)

    def query_volume(self, query_fn, device='cuda:0'):
        """The device volume f32 [1,nx,ny,nz] of query_fn's last channel on the lattice, filled
        in points_batch_size chunks (mesher.py:186-196 without the host copy) -> (volume, axes)."""
        xyz = self.get_grid_uniform(self.config.resolution)['xyz']
        nx, ny, nz = (len(a) for a in xyz)
        n = nx * ny * nz
        vol = torch.empty(n, dtype=torch.float32, device=device)
        bs = self.config.points_batch_size
        for s in range(0, n, bs):
            c = min(bs, n - s)
            pts = self.grid_points(xyz, s, c, device)
            vol[s:s + c] = self.eval_points(pts, query_fn, self.bounding_box, device)[:, -1]
        return vol.view(1, nx, ny, nz), xyz

    def extract(self, volume, xyz):
        """Marching cubes at level_set in world coordinates: verts * spacing + (x0, y0, z0)
        with spacing x[2] - x[1] (mesher.py:206-238)."""
        spacing = [a[2] - a[1] for a in xyz]
        return marching_cubes(volume, self.config.level_set, spacing, shift=[a[0] for a in xyz])

    def vertex_colors(self, verts, color_func, device='cuda:0'):
        """mesher.py:240-253 -> u8 [V,3] on the device.  Co-SLAM's color_func returns [N,1,3]
        (reference quirk); the colours are written as [N,3]."""
        z = [self.eval_points(pnts, color_func, self.bounding_box, device)[..., :3].reshape(-1, 3)
             for pnts in torch.split(verts, self.config.points_batch_size, dim=0)]
        return colors_to_u8(torch.cat(z, 0))

    def get_mesh(self, keyframe_graph, query_fn, color_func=None, device='cuda:0', use_mask=False):
        """mesher.py:179-264 -> TriMesh, or None when nothing crosses level_set."""
        if use_mask:
            raise NotImplementedError('use_mask needs the open3d convex hull of the keyframes '
                                      '(get_bound_from_frames), which is not built')
        with torch.no_grad():
            volume, xyz = self.query_volume(query_fn, device)
            verts, faces = self.extract(volume, xyz)
            if verts.shape[0] == 0:
                print('marching_cubes: no surface extracted from the level set.')
                return None
            colors = None
            if color_func is not None:
                colors = self.vertex_colors(verts, color_func, device).cpu().numpy()
            vertices = verts.cpu().numpy()
            vertices /= self.scale
            return TriMesh(vertices, faces.cpu().numpy(), vertex_colors=colors)
