"""Vox-Fusion algorithm (host-side mirror of slam/algorithms/voxfusion.py): octree growth
from every valid depth pixel of the mapping frame, per-frame pixel sampling -- around the
CUDA march + render step in sparse_voxel.py."""
from __future__ import annotations

import functools
from dataclasses import dataclass, field
from typing import Any, Dict, Type

import numpy as np
import torch

from .algorithm import Algorithm, AlgorithmConfig
from .common import get_camera_rays
from .optimizers import AdamOptimizerConfig
from .sparse_voxel import SparseVoxelConfig


def _vox_optimizers():
    """slam/configs/input_config.py:178-195."""
    A = AdamOptimizerConfig
    return {
        'decoder': {'optimizer': A(lr=5e-3), 'scheduler': None},
        'embeddings': {'optimizer': A(lr=5e-3), 'scheduler': None},
        'tracking_pose': {'optimizer': A(lr=1e-2), 'scheduler': None},
        'mapping_pose': {'optimizer': A(lr=1e-3), 'scheduler': None},
    }


@dataclass
class VoxFusionConfig(AlgorithmConfig):
    """voxfusion.py:18-28 + the vox-fusion entry of input_config.py:159-201."""
    _target: Type = field(default_factory=lambda: VoxFusion)
    model: SparseVoxelConfig = field(default_factory=SparseVoxelConfig)
    keyframe_selection_method: str = 'random'
    tracking_n_iters: int = 30
    mapping_n_iters: int = 15
    mapping_first_n_iters: int = 30
    mapping_window_size: int = 5
    mapping_sample: int = 1024
    min_sample_pixels: int = 100
    tracking_sample: int = 1024
    ray_batch_size: int = 3000
    optimizers: Dict[str, Any] = field(default_factory=_vox_optimizers)


class VoxFusion(Algorithm):
    config: VoxFusionConfig

    def __init__(self, config: VoxFusionConfig, camera, device: str) -> None:
        super().__init__(config, camera, device)
        self.model = self.config.model.setup(camera=camera, bounding_box=None)
        self.model.to(device)
        # voxfusion.py:38-52 precompute: camera-frame directions of every pixel (resident)
        self.rays_d = get_camera_rays(camera.height, camera.width, camera.fx, camera.fy,
                                      camera.cx, camera.cy).float().to(device)
        self.bundle_adjust = True

    # voxfusion.py:55-94
    def get_model_input(self, optimize_frames, is_mapping):
        n = self.config.mapping_sample if is_mapping else self.config.tracking_sample
        rays_o, rays_d, gt_depth, gt_color = self._sample_window(optimize_frames, n)
        return {'rays_o': rays_o, 'rays_d': rays_d, 'target_s': gt_color, 'target_d': gt_depth}

    # voxfusion.py:96-106
    def create_voxels(self, frame):
        depth = self._frame_tensor(frame, 'depth')
        points = (self.rays_d * depth[..., None])[depth > 0].reshape(-1, 3)
        pose = frame.get_pose().detach().to(self.device)
        points = points @ pose[:3, :3].transpose(-1, -2) + pose[:3, 3]
        self.model.insert_points(points)

    def pre_precessing(self, cur_frame, is_mapping):
        if is_mapping:
            self.create_voxels(cur_frame)

    def get_loss(self, optimize_frames, is_mapping, step=None, n_iters=None, coarse=False):
        self.model.freeze_map_grads = not is_mapping  # tracking optimises the pose only
        model_input = self.get_model_input(optimize_frames, is_mapping)
        model_outputs = self.model(model_input)
        if model_outputs is None:  # no ray hit the map (sparse_voxel.py:197-199)
            raise RuntimeError('no ray intersects the voxel map')
        loss_dict = self.model.get_loss_dict(model_outputs, model_input, is_mapping, step)
        return functools.reduce(torch.add, loss_dict.values())

    def render_img(self, c2w, gt_depth=None, idx=None):
        with self.lock, torch.no_grad():
            return self._render_full(c2w, gt_depth)

    # voxfusion.py:171-176
    def get_mesh(self):
        with self.lock, torch.no_grad():
            return self.extract_mesh(clean_mesh=False, require_color=True, res=8)

    def surface_voxels(self):
        """Surface leaves (voxfusion.py:180-185): node ids i64 [B], voxel rows f32 [B,4] (x, y,
        z, side) and centres f32 [B,3], on the device."""
        model = self.model
        if model._dev_svo is not None:
            voxels, _, features = model._dev_svo.export()
        else:
            voxels, _, features = (t.to(self.device) for t in model.export_octree())
        keep = ~features.eq(-1).any(-1)
        ids = torch.nonzero(keep).squeeze(1)
        return ids, voxels[ids], model.map_states['voxel_center_xyz'][ids]

    @torch.no_grad()
    def extract_mesh(self, res=8, clean_mesh=False, require_color=False):
        """voxfusion.py:178-248 -> TriMesh (None without a surface).  One batched lattice query
        over every surface voxel, one batched marching cubes (vertices are not shared between
        voxels, like the reference's per-voxel meshes), and the vertex -> voxel lookup
        `points // voxel_size == voxels[:, :3]` as a sort + searchsorted over integer keys.
        clean_mesh is a no-op in the reference as well (its TODO)."""
        from .mesher import TriMesh, colors_to_u8, marching_cubes
        if self.model.map_states is None:
            return None
        ids, voxels, centres = self.surface_voxels()
        if ids.numel() == 0:
            return None
        vs = self.model.config.voxel_size
        sdf = self.model.get_scores(ids, res)
        s = 1.0 / (res - 1)
        verts, faces = marching_cubes(sdf, 0.0, (s, s, s), shift=(-0.5,) * 3, scale=(vs,) * 3,
                                      origin=centres)
        if verts.shape[0] == 0:
            return None
        colors = None
        if require_color:
            colors = colors_to_u8(self.vertex_colors(verts, ids, voxels)).cpu().numpy()
        return TriMesh(verts.cpu().numpy(), faces.cpu().numpy(), vertex_colors=colors)

    def vertex_colors(self, verts, ids, voxels):
        """voxfusion.py:205-239: colour f32 [V,3] of each vertex from the surface voxel with
        voxels[:, :3] == verts // voxel_size (a vertex on a voxel face goes to the neighbour
        its floor names), 0 where no surface voxel matches."""
        keys = _voxel_keys(voxels[:, :3])
        order = torch.argsort(keys)
        skeys = keys[order]
        q = _voxel_keys(verts // self.model.config.voxel_size)
        pos = torch.searchsorted(skeys, q).clamp(max=skeys.shape[0] - 1)
        hit = skeys[pos] == q
        rgb = self.model.eval_points(verts, ids[order[pos]])
        return torch.where(hit[:, None], rgb, torch.zeros_like(rgb))


def _voxel_keys(v):
    """int64 key of integer-valued voxel coordinates f32 [N,3] (|coordinate| < 2^20)."""
    k = v.to(torch.int64) + (1 << 20)
    return (k[:, 0] << 42) | (k[:, 1] << 21) | k[:, 2]
