"""Point-SLAM algorithm (host-side mirror of slam/algorithms/point_slam.py): dynamic add /
query radii from the colour gradient, neural-point insertion per mapping frame, frustum
point selection, stage schedule geometry -> color -- around the CUDA step in
conv_onet_pointslam.py.  skimage / scipy / cv2 calls are restated in torch on the device:
  rgb2gray      Y = 0.2125 R + 0.7154 G + 0.0721 B            (skimage.color)
  sobel_h / _v  [1,2,1]^T x [1,0,-1] / 4, mode='reflect'      (skimage.filters)
  interp1d      piecewise linear through 3 knots               (scipy.interpolate)"""
from __future__ import annotations

import functools
from dataclasses import dataclass, field
from typing import Any, Dict, Type

import numpy as np
import torch
import torch.nn.functional as F

from .algorithm import Algorithm, AlgorithmConfig
from .common import get_samples, get_samples_with_pixel_grad
from .conv_onet_pointslam import ConvOnet2Config
from .keyframe_selection import frustum_mask
from .optimizers import AdamOptimizerConfig
from .schedulers import PointSLAMSchedulerConfig


def _point_optimizers():
    """slam/configs/input_config.py:328-375."""
    A, S = AdamOptimizerConfig, PointSLAMSchedulerConfig
    return {
        'decoder': {'optimizer': A(), 'scheduler': S(start_lr=0.001, end_lr=0.005)},
        'geometry': {'optimizer': A(), 'scheduler': S(start_lr=0.03, end_lr=0.005)},
        'color': {'optimizer': A(), 'scheduler': S(start_lr=0.0, end_lr=0.005)},
        'tracking_pose_r': {'optimizer': A(lr=0.002 * 0.2), 'scheduler': None},
        'tracking_pose_t': {'optimizer': A(lr=0.002), 'scheduler': None},
        'mapping_pose_r': {'optimizer': A(lr=0.0002), 'scheduler': None},
        'mapping_pose_t': {'optimizer': A(lr=0.0002), 'scheduler': None},
    }


@dataclass
class PointSLAMConfig(AlgorithmConfig):
    """point_slam.py:20-60 + the point-slam entry of input_config.py:298-380."""
    _target: Type = field(default_factory=lambda: PointSLAM)
    model: ConvOnet2Config = field(default_factory=ConvOnet2Config)
    separate_LR: bool = True
    rot_rep: str = 'axis_angle'
    use_dynamic_radius: bool = True
    pixels_adding: int = 6000
    tracking_n_iters: int = 40
    mapping_n_iters: int = 300
    mapping_first_n_iters: int = 1500
    mapping_window_size: int = 12
    mapping_sample: int = 5000
    min_sample_pixels: int = 40
    tracking_sample: int = 1500
    ray_batch_size: int = 3000
    tracking_sample_with_color_grad: bool = False
    tracking_Wedge: int = 100
    tracking_Hedge: int = 100
    mapping_geo_iter_ratio: float = 0.4
    mapping_pixels_based_on_color_grad: int = 1000
    mapping_frustum_feature_selection: bool = True
    mapping_frustum_edge: int = -4
    mapping_BA: bool = False
    model_encode_exposure: bool = False
    pointcloud_radius_add_max: float = 0.08
    pointcloud_radius_add_min: float = 0.02
    pointcloud_radius_add: float = 0.04
    pointcloud_radius_query: float = 0.08
    pointcloud_radius_query_ratio: int = 2
    pointcloud_color_grad_threshold: float = 0.15
    clean_mesh: bool = True
    optimizers: Dict[str, Any] = field(default_factory=_point_optimizers)


def sobel_magnitude(rgb):
    """sqrt(sobel_v^2 + sobel_h^2) of rgb2gray(rgb) (float64, like skimage)."""
    img = rgb.double()
    gray = 0.2125 * img[..., 0] + 0.7154 * img[..., 1] + 0.0721 * img[..., 2]
    g = F.pad(gray[None, None], (1, 1, 1, 1), mode='replicate')  # scipy 'reflect' = edge repeat
    sm = torch.tensor([1., 2., 1.], dtype=torch.float64, device=img.device)
    df = torch.tensor([1., 0., -1.], dtype=torch.float64, device=img.device)
    kh = (df[:, None] * sm[None, :] / 4.0)[None, None]  # horizontal edges: derivative along rows
    kv = (sm[:, None] * df[None, :] / 4.0)[None, None]
    # scipy.ndimage.convolve flips the kernel; conv2d is a correlation -> flip back
    gh = F.conv2d(g, torch.flip(kh, (2, 3)))[0, 0]
    gv = F.conv2d(g, torch.flip(kv, (2, 3)))[0, 0]
    return torch.sqrt(gv**2 + gh**2)


class PointSLAM(Algorithm):
    config: PointSLAMConfig

    def __init__(self, config: PointSLAMConfig, camera, device: str) -> None:
        super().__init__(config, camera, device)
        self.stage = 'color'
        mc = self.config.model
        mc.model_encode_exposure = self.config.model_encode_exposure
        mc.use_dynamic_radius = self.config.use_dynamic_radius
        mc.mapping_pixels_based_on_color_grad = self.config.mapping_pixels_based_on_color_grad
        self.model = mc.setup(camera=camera)
        self.model.to(device)
        self.dynamic_r_query_allkeyframe = {}

    # point_slam.py:339-366
    def cal_dynamic_radius(self, rgb):
        cfg = self.config
        thr = cfg.pointcloud_color_grad_threshold
        mag = torch.clamp(sobel_magnitude(torch.as_tensor(np.asarray(rgb)).to(self.device)), 0.0, thr)
        rmax, rmin = cfg.pointcloud_radius_add_max, cfg.pointcloud_radius_add_min
        # interp1d([0, 0.01, thr], [rmax, rmax, rmin])
        r_add = torch.where(mag <= 0.01, torch.full_like(mag, rmax),
                            rmax + (mag - 0.01) * (rmin - rmax) / (thr - 0.01))
        return r_add, cfg.pointcloud_radius_query_ratio * r_add

    # point_slam.py:81-155
    def pre_precessing(self, cur_frame, is_mapping):
        cfg = self.config
        c2w = cur_frame.get_pose()
        key = str(int(cur_frame.fid))
        r_add = None
        if cfg.use_dynamic_radius:
            r_add, r_query = self.cal_dynamic_radius(cur_frame.rgb)
            self.dynamic_r_query_allkeyframe[key] = r_query
        if not is_mapping:
            return
        depth = self._frame_tensor(cur_frame, 'depth')
        rgb = self._frame_tensor(cur_frame, 'rgb')
        n_add = cfg.pixels_adding
        if cur_frame.fid == 0:
            n_add = int(torch.clamp(cfg.pixels_adding * ((depth.median() / 2.5)**2),
                                    min=cfg.pixels_adding, max=cfg.pixels_adding * 3).int())
        ro, rd, d, c, i, j = get_samples(self.camera, n_add, c2w, depth, rgb, device=self.device,
                                         depth_filter=True, return_index=True)
        npc = self.model.model_update(self.device)
        npc.add_neural_points(ro.detach(), rd.detach(), d, c,
                              dynamic_radius=r_add[j, i] if r_add is not None else None)
        if cfg.mapping_pixels_based_on_color_grad > 0:
            # point_slam.py:124-142: a second insertion pass over the pixels with the largest
            # colour gradient, searched with the (smaller) per-pixel add radius / radius_min
            ro_g, rd_g, d_g, c_g, i_g, j_g = get_samples_with_pixel_grad(
                self.camera, cfg.mapping_pixels_based_on_color_grad, c2w, cur_frame.depth,
                cur_frame.rgb, device=self.device, depth_filter=True, return_index=True)
            npc.add_neural_points(ro_g.detach(), rd_g.detach(), d_g, c_g, is_pts_grad=True,
                                  dynamic_radius=r_add[j_g, i_g] if r_add is not None else None)
        if cfg.mapping_frustum_feature_selection and npc.pts_num() > 0:
            m = frustum_mask(self.camera, c2w.detach(), npc.cloud_pos(), cur_frame.depth,
                             edge=cfg.mapping_frustum_edge)
            npc.set_mask(m)

    # point_slam.py:157-165
    def optimizer_config_update(self, max_iters, coarse=False):
        self.bundle_adjust = len(self.keyframe_graph) > 4 and self.config.mapping_BA
        for _, params in self.config.optimizers.items():
            if params['scheduler'] is not None:
                params['optimizer'].lr = 1.0
                params['scheduler'].max_steps = max_iters
                params['scheduler'].geo_iter_ratio = self.config.mapping_geo_iter_ratio

    # point_slam.py:167-249
    def get_model_input(self, optimize_frames, is_mapping):
        cfg = self.config
        n, Hedge, Wedge = cfg.tracking_sample, cfg.tracking_Hedge, cfg.tracking_Wedge
        if is_mapping:
            n = int(np.maximum(cfg.mapping_sample // len(optimize_frames), cfg.min_sample_pixels))
            Hedge = Wedge = 0
        if not is_mapping and cfg.tracking_sample_with_color_grad:
            # point_slam.py:192-205: tracking pixels by colour gradient (per frame, host draw)
            parts = [get_samples_with_pixel_grad(self.camera, n, f.get_pose(), f.depth, f.rgb,
                                                 device=self.device, Hedge=Hedge, Wedge=Wedge,
                                                 depth_filter=True, return_index=True)
                     for f in optimize_frames]
            rays_o, rays_d = torch.cat([p[0] for p in parts]), torch.cat([p[1] for p in parts])
            gt_depth = torch.cat([p[2] for p in parts]).reshape(-1, 1)
            gt_color = torch.cat([p[3] for p in parts])
            i, j = torch.cat([p[4] for p in parts]), torch.cat([p[5] for p in parts])
            fidx = torch.cat([torch.full((p[0].shape[0],), k, device=self.device)
                              for k, p in enumerate(parts)])
        else:
            rays_o, rays_d, gt_depth, gt_color, i, j = self._sample_window(
                optimize_frames, n, Hedge, Wedge, return_index=True)
            fidx = torch.arange(len(optimize_frames), device=self.device).repeat_interleave(n)
        r_query = None
        if cfg.use_dynamic_radius:
            maps = torch.stack([self.dynamic_r_query_allkeyframe[str(int(f.fid))]
                                for f in optimize_frames])  # [F,H,W]
            r_query = maps[fidx, j, i]
        with torch.no_grad():
            d = gt_depth.squeeze(-1)
            valid = d > 0  # per-frame depth_filter=True of get_samples (common.py:214-221)
            dv = d[valid]
            # outlier filter on the depth-filtered batch (Q9: batch-global median / max)
            keep = (valid & (d <= torch.minimum(10 * dv.median(), 1.2 * torch.max(dv)))
                    ).nonzero().squeeze(1)
        sel = lambda x: x.index_select(0, keep)
        return {'rays_o': sel(rays_o), 'rays_d': sel(rays_d), 'target_s': sel(gt_color),
                'target_d': sel(gt_depth),
                'batch_dynamic_r': sel(r_query) if r_query is not None else None,
                'stage': self.stage, 'is_mapping': is_mapping}

    def set_stage(self, is_mapping, step, n_iters):
        if not is_mapping:
            self.stage = 'color'
        elif step <= int(n_iters * self.config.mapping_geo_iter_ratio):
            self.stage = 'geometry'
        else:
            self.stage = 'color'

    def get_loss(self, optimize_frames, is_mapping, step, n_iters, coarse=False):
        self.set_stage(is_mapping, step, n_iters)
        self.model.freeze_map_grads = not is_mapping  # tracking optimises the pose only
        model_input = self.get_model_input(optimize_frames, is_mapping)
        model_outputs = self.model(model_input)
        loss_dict = self.model.get_loss_dict(model_outputs, model_input, is_mapping, self.stage)
        return functools.reduce(torch.add, loss_dict.values())

    def render_img(self, c2w, gt_depth=None, idx=None):
        with self.lock, torch.no_grad():
            per_pixel = None
            if self.config.use_dynamic_radius:
                per_pixel = {'batch_dynamic_r':
                             self.dynamic_r_query_allkeyframe[str(int(idx))].reshape(-1).float()}
            return self._render_full(c2w, gt_depth, extra={'stage': 'color'}, per_pixel=per_pixel)

    # point_slam.py:426-435
    def get_mesh(self):
        """TSDF fusion of the keyframes (common.get_mesh_from_RGBD), cleaned with clean_mesh
        when config.clean_mesh (vertices, faces, uint8 colours) or else vertices and faces only,
        as the reference's Trimesh(vertices, faces).  None without keyframes or surface."""
        from .common import clean_mesh, get_mesh_from_RGBD
        from .mesher import TriMesh
        with self.lock, torch.no_grad():
            if not self.keyframe_graph:
                return None
            mesh = get_mesh_from_RGBD(self.camera, self.keyframe_graph,
                                      frame_tensor=self._frame_tensor)
            if mesh.faces.shape[0] == 0:
                return None
            if self.config.clean_mesh:
                mesh = clean_mesh(mesh)
                if mesh.faces.shape[0] == 0:
                    return None
            else:
                mesh = TriMesh(mesh.vertices.cpu().numpy(), mesh.faces.cpu().numpy())
            self.cur_mesh = mesh
            return mesh
