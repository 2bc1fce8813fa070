"""Restatement of Point-SLAM's rendering_sample_near_pcl: the samples of rays without depth
placed near the neural point cloud, and the step that renders with them.

ORACLE / TEST INFRASTRUCTURE -- never imported by xrdslam_b200/.

Follows (reference @ f0366f20):
  slam/model_components/neural_point_cloud.py:284-348  NeuralPointCloud.sample_near_pcl
  slam/models/conv_onet_pointslam.py:379-409, 450-451  render_batch_ray with the option on
with faiss replaced by exact search, as everywhere in oracle/pointslam.py (SURVEY A.4).
Pinned against the reference's own functions by tests/test_pointslam_near_pcl_cpu.py.

For a batch with depth gt_d and far = min(5 mean(gt_d), max(1.2 gt_d)) (10 without depth):
  1. Z = rays with !(gt_d > 0) (NaN included);
  2. 25 march depths zq = torch.linspace(near_end, far, 25) in f32, points o + d * zq;
  3. a march point hits when some cloud point lies at f32 squared distance
     ((dx^2 + dy^2) + dz^2) < f32(radius_query ** 2)  (the FIXED query radius);
  4. a ray is invalid with fewer than two hits;
  5. valid: z = f32(np.linspace(sec[c0], sec[c1], num)), sec = np.linspace(near_end, far, 25),
     c0 / c1 the first and SECOND hit;
  6. invalid: z = f32(np.linspace(near_end, far, num)) in float64;
  7. valid_ray_mask &= !(Z and invalid); the rendered depth of Z is not zeroed.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle.pointslam import PointOracle

MARCH = 25


def linspace_f32(start, end, n):
    """torch.linspace(start, end, n) in float32: torch's two-sided formula."""
    start, end = np.float32(start), np.float32(end)
    step = np.float32((end - start) / np.float32(n - 1))
    k = np.arange(n)
    lo = start + step * k.astype(np.float32)
    hi = end - step * (n - 1 - k).astype(np.float32)
    return np.where(k < n // 2, lo, hi).astype(np.float32)


def linspace_f64(start, stop, n):
    """np.linspace(start, stop, n) restated: arange * step + start (or, where the step
    underflows to 0, arange / div * delta + start), the last element set to stop."""
    start, stop = float(start), float(stop)
    div = float(n - 1)
    delta = stop - start
    step = delta / div
    k = np.arange(n, dtype=np.float64)
    y = (k / div) * delta if step == 0 else k * step
    y = y + start
    y[-1] = stop
    return y


def march_hits(cloud, pts, radius_query, chunk_elems=1 << 24):
    """[Q] bool: some cloud point at f32 squared distance < f32(radius_query ** 2)."""
    r2 = torch.tensor(np.float32(radius_query ** 2))
    out = torch.zeros(pts.shape[0], dtype=torch.bool)
    N = cloud.shape[0]
    if N == 0:
        return out
    step = max(1, chunk_elems // N)
    for s in range(0, pts.shape[0], step):
        d = cloud[None, :, :] - pts[s:s + step, None, :]
        D = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
        out[s:s + step] = (D < r2).any(1)
    return out


def sample_near_pcl(cloud, rays_o, rays_d, target_d, far, near_end, num, radius_query):
    """Steps 1-6 for every ray -> (z [R,num] f32, near [R] bool).  Rows of rays with depth are
    zero in z and True in near (the step takes their samples from the surface)."""
    ro = rays_o.detach().float().reshape(-1, 3)
    rd = rays_d.detach().float().reshape(-1, 3)
    R = ro.shape[0]
    Z = ~(target_d.detach().float().reshape(-1) > 0)
    far32 = np.float32(float(far))
    zq = torch.from_numpy(linspace_f32(near_end, far32, MARCH))
    pts = (ro[:, None, :] + rd[:, None, :] * zq[None, :, None]).reshape(-1, 3)
    hits = march_hits(cloud.detach().float(), pts, radius_query).reshape(R, MARCH)
    sec = linspace_f64(near_end, float(far32), MARCH)
    off = linspace_f64(near_end, float(far32), num)
    z = np.zeros((R, num), np.float64)
    near = np.ones(R, bool)
    for r in torch.nonzero(Z).flatten().tolist():
        c = torch.nonzero(hits[r]).flatten().tolist()
        if len(c) >= 2:
            z[r] = linspace_f64(sec[c[0]], sec[c[1]], num)
        else:
            z[r] = off
            near[r] = False
    return torch.from_numpy(z).float(), torch.from_numpy(near)


def far_of(target_d, R):
    """render_batch_ray's batch-global far (conv_onet_pointslam.py:336-354) as f32."""
    if target_d is None:
        return torch.tensor(10.0)
    gt = target_d.detach().float().reshape(-1)
    return torch.minimum(5 * gt.mean(), torch.max(gt * 1.2)).float()


class NearPclOracle(PointOracle):
    """PointOracle with rendering_sample_near_pcl on (step 7 on top of PointOracle.render)."""
    radius_query = 0.08

    def render(self, rays_o, rays_d, target_d, radius, rand_feat, stage='geometry',
               rand_feat_color=None):
        R = rays_o.shape[0]
        far = far_of(target_d, R)
        td = torch.zeros(R, 1) if target_d is None else target_d
        self._near_pcl = sample_near_pcl(self.cloud, rays_o, rays_d, td, far, self.near_end,
                                         self.n_surface, self.radius_query)
        out = super().render(rays_o, rays_d, td, radius, rand_feat, stage, rand_feat_color)
        out['valid_ray_mask'] = out['valid_ray_mask'] & self._near_pcl[1]
        return out

    def sample_z(self, target_d):
        z, nz = super().sample_z(target_d)
        zn, _ = self._near_pcl
        z = torch.where(nz[:, None], z, zn)
        return z, torch.ones_like(nz)  # the depth of zero-depth rays is kept
