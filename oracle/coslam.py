"""Torch-CPU restatement of the Co-SLAM render-and-optimise step.

ORACLE / TEST INFRASTRUCTURE -- never imported by xrdslam_b200/.

Follows (reference @ f0366f20, paths relative to /root/reference):
  slam/models/joint_encoding.py:250-344   render_rays   (sampling, perturb, pts)
  slam/models/joint_encoding.py:483-507   run_network   (f64 bbox normalisation)
  slam/models/joint_encoding.py:463-481   query_color_sdf
  slam/model_components/decoder_coslam.py:139-163  ColorSDFNet_v2
  slam/models/joint_encoding.py:346-406   sdf2weights / raw2outputs
  slam/models/joint_encoding.py:94-147    get_loss_dict
  slam/model_components/utils.py:100-186  get_masks / compute_loss / get_sdf_loss
  slam/models/joint_encoding.py:165-197   smoothness
Pinned against the reference's own JointEncoding class (run on CPU through
oracle/ref_harness.py) by tests/test_oracle_vs_reference.py and by the committed
fixtures in tests/golden/coslam_*.npz.  The tinycudann encodings inside are
restated (oracle/tcnn_restated.py) -> "parity unpinned" at that boundary.

Randomness is an explicit input: ``noise`` [R,S] replaces
``torch.rand(z_vals.shape)`` (joint_encoding.py:292) and ``smooth_rand`` [2,3]
replaces the two torch.rand calls in smoothness (:176,:179-181).
"""
from __future__ import annotations

from dataclasses import dataclass

import torch
import torch.nn.functional as F

from oracle.tcnn_restated import HashGridRestated, OneBlobRestated


@dataclass
class CoslamCfg:
    # joint_encoding.py:18-66 defaults, overridden as in input_config.py:253-254
    voxel_sdf: float = 0.02
    pos_nbins: int = 16
    hashsize: int = 16
    geo_feat_dim: int = 15
    hidden_dim: int = 32
    hidden_dim_color: int = 32
    rgb_weight: float = 5.0
    depth_weight: float = 0.1
    sdf_weight: float = 1000.0
    fs_weight: float = 10.0
    smooth_weight: float = 1e-6
    smooth_pts: int = 32
    smooth_vox: float = 0.1
    smooth_margin: float = 0.05
    n_samples: int = 256
    n_sample_d: int = 32
    range_d: float = 0.1
    n_range_d: int = 11
    perturb: int = 1
    trunc: float = 0.1
    rgb_missing: float = 0.05
    sc_factor: int = 1
    near: float = 0.0
    far: float = 5.0
    depth_trunc: float = 100.0


class CoslamOracle(torch.nn.Module):
    def __init__(self, bounding_box, cfg: CoslamCfg = None):
        super().__init__()
        self.cfg = cfg or CoslamCfg()
        c = self.cfg
        self.bounding_box = torch.as_tensor(bounding_box, dtype=torch.float64)
        # get_resolution (:199-210) / get_encoder (encodings_coslam.py:39-53)
        dim_max = (self.bounding_box[:, 1] - self.bounding_box[:, 0]).max()
        self.resolution_sdf = int(dim_max / c.voxel_sdf)
        import numpy as np
        pls = np.exp2(np.log2(self.resolution_sdf / 16) / (16 - 1))
        self.embed_fn = HashGridRestated(3, 16, 2, c.hashsize, 16, pls)
        self.embedpos_fn = OneBlobRestated(3, c.pos_nbins)
        in_sdf = 32 + 3 * c.pos_nbins
        in_col = 3 * c.pos_nbins + c.geo_feat_dim
        L = torch.nn.Linear
        self.sdf0 = L(in_sdf, c.hidden_dim, bias=False)
        self.sdf1 = L(c.hidden_dim, 1 + c.geo_feat_dim, bias=False)
        self.col0 = L(in_col, c.hidden_dim_color, bias=False)
        self.col1 = L(c.hidden_dim_color, 3, bias=False)

    # ---- sampling -----------------------------------------------------------
    def sample_z(self, n_rays, target_d, noise):
        c = self.cfg
        if target_d is not None:
            z_samples = torch.linspace(-c.range_d, c.range_d,
                                       steps=c.n_range_d).to(target_d)
            z_samples = z_samples[None, :].repeat(n_rays, 1) + target_d
            z_samples[target_d.squeeze(-1) <= 0] = torch.linspace(
                c.near, c.far, steps=c.n_range_d).to(target_d)
            z_vals = torch.linspace(c.near, c.far,
                                    c.n_sample_d)[None, :].repeat(n_rays, 1).to(target_d.device)
            z_vals, _ = torch.sort(torch.cat([z_vals, z_samples], -1), -1)
        else:
            z_vals = torch.linspace(c.near, c.far,
                                    c.n_samples)[None, :].repeat(n_rays, 1)
        if c.perturb > 0:
            mids = .5 * (z_vals[..., 1:] + z_vals[..., :-1])
            upper = torch.cat([mids, z_vals[..., -1:]], -1)
            lower = torch.cat([z_vals[..., :1], mids], -1)
            z_vals = lower + (upper - lower) * noise
        return z_vals

    # ---- network ------------------------------------------------------------
    def normalise(self, pts_flat):
        bb = self.bounding_box.to(pts_flat.device)
        return (pts_flat - bb[:, 0]) / (bb[:, 1] - bb[:, 0])  # f64 (C2)

    def query_color_sdf(self, x_norm):
        embed = self.embed_fn(x_norm)
        pos = self.embedpos_fn(x_norm)
        h = self.sdf1(F.relu(self.sdf0(torch.cat([embed, pos], -1))))
        sdf, geo = h[..., :1], h[..., 1:]
        rgb = self.col1(F.relu(self.col0(torch.cat([pos, geo], -1))))
        return torch.cat([rgb, sdf], -1)

    def sdf2weights(self, sdf, z_vals):
        tr = self.cfg.trunc
        weights = torch.sigmoid(sdf / tr) * torch.sigmoid(-sdf / tr)
        signs = sdf[:, 1:] * sdf[:, :-1]
        mask = torch.where(signs < 0.0, torch.ones_like(signs),
                           torch.zeros_like(signs))
        inds = torch.argmax(mask, dim=1)[..., None]
        z_min = torch.gather(z_vals, 1, inds)
        mask = torch.where(z_vals < z_min + self.cfg.sc_factor * tr,
                           torch.ones_like(z_vals), torch.zeros_like(z_vals))
        weights = weights * mask
        return weights / (torch.sum(weights, dim=-1, keepdim=True) + 1e-8)

    def render_rays(self, rays_o, rays_d, target_d, noise):
        n_rays = rays_o.shape[0]
        z_vals = self.sample_z(n_rays, target_d, noise).to(rays_o)
        pts = rays_o[..., None, :] + rays_d[..., None, :] * z_vals[..., :, None]
        flat = pts.reshape(-1, 3)
        raw = self.query_color_sdf(self.normalise(flat)).reshape(
            n_rays, -1, 4)
        rgb = torch.sigmoid(raw[..., :3])
        weights = self.sdf2weights(raw[..., 3], z_vals)
        rgb_map = torch.sum(weights[..., None] * rgb, -2)
        depth_map = torch.sum(weights * z_vals, -1)
        depth_var = torch.sum(
            weights * torch.square(z_vals - depth_map.unsqueeze(-1)), dim=-1)
        disp_map = 1. / torch.max(1e-10 * torch.ones_like(depth_map),
                                  depth_map / torch.sum(weights, -1))
        acc_map = torch.sum(weights, -1)
        return dict(rgb=rgb_map, depth=depth_map, disp_map=disp_map,
                    acc_map=acc_map, depth_var=depth_var, z_vals=z_vals,
                    raw=raw, weights=weights)

    # ---- losses -------------------------------------------------------------
    def loss_dict(self, out, target_s, target_d, is_mapping, first,
                  smooth_rand=None):
        c = self.cfg
        valid = (target_d.squeeze(-1) > 0.) * (target_d.squeeze(-1) <
                                               c.depth_trunc)
        # Q1: rgb_weight is a bool tensor -> every ray weighs 1
        rgb_loss = F.mse_loss(out['rgb'], target_s)
        depth_loss = F.mse_loss(out['depth'][valid],
                                target_d.squeeze(-1)[valid])
        z_vals, sdf = out['z_vals'], out['raw'][..., -1]
        tr = c.trunc * c.sc_factor
        front = torch.where(z_vals < (target_d - tr), torch.ones_like(z_vals),
                            torch.zeros_like(z_vals))
        back = torch.where(z_vals > (target_d + tr), torch.ones_like(z_vals),
                           torch.zeros_like(z_vals))
        dmask = torch.where(target_d > 0.0, torch.ones_like(target_d),
                            torch.zeros_like(target_d))
        sdf_mask = (1.0 - front) * (1.0 - back) * dmask
        n_fs = torch.count_nonzero(front)
        n_sdf = torch.count_nonzero(sdf_mask)
        n = n_sdf + n_fs
        fs_w = 1.0 - n_fs / n
        sdf_w = 1.0 - n_sdf / n
        fs_loss = F.mse_loss(sdf * front, torch.ones_like(sdf) * front) * fs_w
        sdf_loss = F.mse_loss((z_vals + sdf * tr) * sdf_mask,
                              target_d * sdf_mask) * sdf_w
        d = {
            'rgb_loss': rgb_loss * c.rgb_weight,
            'depth_loss': depth_loss * c.depth_weight,
            'sdf_loss': sdf_loss * c.sdf_weight,
            'fs_loss': fs_loss * c.fs_weight,
        }
        if is_mapping and not first:
            d['smooth_loss'] = self.smoothness(smooth_rand) * c.smooth_weight
        return d

    def smooth_points(self, smooth_rand, sample_points=None, voxel=None, margin=None):
        """pts (f64, normalised) of the smoothness lattice; smooth_rand[0] is
        torch.rand(3) of :176, smooth_rand[1] the torch.rand((1,1,1,3)) of :179.
        sample_points / voxel / margin default to the config's."""
        c = self.cfg
        sp = c.smooth_pts if sample_points is None else sample_points
        vox = c.smooth_vox if voxel is None else voxel
        margin = c.smooth_margin if margin is None else margin
        bb = self.bounding_box.to(self.embed_fn.params.device)
        smooth_rand = smooth_rand.to(bb.device)
        n = sp - 1
        grid_size = (sp - 1) * vox
        offset_max = bb[:, 1] - bb[:, 0] - grid_size - 2 * margin
        offset = smooth_rand[0].to(offset_max) * offset_max + margin
        ar = torch.arange(0, n, dtype=torch.long, device=bb.device)
        x, y, z = torch.meshgrid(ar, ar, ar, indexing='ij')
        coords = torch.stack([x, y, z], -1).float().to(bb)
        pts = (coords + smooth_rand[1].reshape(1, 1, 1, 3).to(bb)
               ) * vox + bb[:, 0] + offset
        return (pts - bb[:, 0]) / (bb[:, 1] - bb[:, 0])

    def smoothness(self, smooth_rand):
        c = self.cfg
        p = self.smooth_points(smooth_rand)
        feat = self.embed_fn(p.reshape(-1, 3)).reshape(*p.shape[:-1], -1)
        tv_x = torch.pow(feat[1:, ...] - feat[:-1, ...], 2).sum()
        tv_y = torch.pow(feat[:, 1:, ...] - feat[:, :-1, ...], 2).sum()
        tv_z = torch.pow(feat[:, :, 1:, ...] - feat[:, :, :-1, ...], 2).sum()
        return (tv_x + tv_y + tv_z) / (c.smooth_pts**3)

    # ---- one full step ------------------------------------------------------
    def step(self, rays_o, rays_d, target_s, target_d, noise, is_mapping,
             first, smooth_rand=None):
        out = self.render_rays(rays_o, rays_d, target_d, noise)
        ld = self.loss_dict(out, target_s, target_d, is_mapping, first,
                            smooth_rand)
        total = None
        for v in ld.values():
            total = v if total is None else total + v
        return out, ld, total
