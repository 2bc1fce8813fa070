"""Neural point cloud of Point-SLAM, H100-native (host-side mirror of
slam/model_components/neural_point_cloud.py): positions and features are device tensors (the
reference keeps positions in Python lists and re-tensorises them every call,
decoder_pointslam.py:172,417), and neighbour search is an EXACT radius-limited 8-NN over a
uniform hash grid (csrc/pointslam.cu) instead of faiss-gpu IVFFlat (approximate, un-vendored;
SURVEY A.4).  faiss's sentinels are kept: missing neighbour -> id -1, D = FLT_MAX."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch
import torch.nn as nn

from . import _cabi
from ._cabi import XrdPointIndex, ptr


class NeuralPointCloud(nn.Module):
    def __init__(self, c_dim=32, nn_num=8, radius_add=0.04, radius_min=0.02, radius_query=0.08,
                 n_add=3, near_end_surface=0.98, far_end_surface=1.02, device='cuda:0',
                 cell=0.08, log2_table=20):
        super().__init__()
        self.c_dim, self.nn_num = c_dim, nn_num
        self.radius_add, self.radius_min, self.radius_query = radius_add, radius_min, radius_query
        self.N_add = n_add
        self.near_end_surface, self.far_end_surface = near_end_surface, far_end_surface
        self.device = torch.device(device)
        self.cell = float(np.float32(cell))
        self.table_size = 1 << log2_table
        self._pos = torch.zeros(0, 3, device=self.device)
        self.geo_feats = None
        self.col_feats = None
        self.frustum_mask = None
        self._index = None

    # ---- container -----------------------------------------------------------
    def pts_num(self):
        return self._pos.shape[0]

    def cloud_pos(self, index=None):
        return self._pos if index is None else self._pos[index]

    def set_mask(self, new_mask):
        self.frustum_mask = new_mask.reshape(-1).to(self.device).to(torch.uint8).contiguous()

    def set_cloud(self, pos, geo_feats, col_feats=None):
        """Replace the whole cloud (checkpoint restore / parity tests)."""
        dev = self.device
        self._pos = pos.detach().to(dev, torch.float32).contiguous()
        self.geo_feats = nn.Parameter(geo_feats.detach().to(dev, torch.float32).contiguous())
        if col_feats is None:
            col_feats = torch.zeros_like(self.geo_feats)
        self.col_feats = nn.Parameter(col_feats.detach().to(dev, torch.float32).contiguous())
        self.frustum_mask = torch.ones(self._pos.shape[0], dtype=torch.uint8, device=dev)
        self._index = None

    def get_geo_feats(self):
        return self.geo_feats

    # ---- index ----------------------------------------------------------------
    def rebuild_index(self):
        """Bucket = hash(floor(x / cell)) as in csrc/pointslam.cu:bucket_of; built on the device
        by xrd_pointslam_knn_build (histogram, scan, scatter, per-bucket id sort)."""
        N = self._pos.shape[0]
        dev = self.device
        i32 = dict(dtype=torch.int32, device=dev)
        start, end = torch.empty(self.table_size, **i32), torch.empty(self.table_size, **i32)
        ids = torch.empty(max(N, 1), **i32)
        ws, nb = _cabi.workspace(dev, 'pointslam_knn_build', self.table_size)
        _cabi.launch_on(dev, 'xrd_pointslam_knn_build', ptr(self._pos), N, self.cell,
                        self.table_size, ptr(start), ptr(end), ptr(ids), ptr(ws), nb)
        self._index = dict(sorted_ids=ids, cell_start=start, cell_end=end, n=N)

    def rebuild_index_torch(self):
        """The same index with torch ops (stable argsort of the bucket keys): the reference
        the device build is tested against."""
        N = self._pos.shape[0]
        inv = float(np.float32(1.0) / np.float32(self.cell))
        ijk = torch.floor(self._pos * inv).to(torch.int64)
        M = 0xFFFFFFFF
        h = ((ijk[:, 0] * 73856093) & M) ^ ((ijk[:, 1] * 19349663) & M) ^ ((ijk[:, 2] * 83492791) & M)
        key = (h & (self.table_size - 1)).to(torch.int64)
        order = torch.argsort(key, stable=True)
        skey = key[order]
        counts = torch.bincount(skey, minlength=self.table_size)
        end = torch.cumsum(counts, 0)
        return dict(sorted_ids=order.to(torch.int32).contiguous(),
                    cell_start=(end - counts).to(torch.int32).contiguous(),
                    cell_end=end.to(torch.int32).contiguous(), n=N)

    def index_struct(self):
        if self._index is None or self._index['n'] != self._pos.shape[0]:
            self.rebuild_index()
        ix = self._index
        return XrdPointIndex(ptr(self._pos), self._pos.shape[0], self.cell, self.table_size,
                             ptr(ix['cell_start']), ptr(ix['cell_end']), ptr(ix['sorted_ids']))

    def find_neighbors(self, pos, radius):
        """-> D [P,8] squared distances, I [P,8] int32 ids, neighbor_num [P]
        (neural_point_cloud.py:223-282 semantics; radius: float or per-point tensor)."""
        pos = pos.detach().to(self.device, torch.float32).contiguous()
        P = pos.shape[0]
        if not torch.is_tensor(radius):
            radius = torch.full((1,), float(radius), device=self.device)
            stride = 0
        else:
            radius = radius.to(self.device, torch.float32).reshape(-1).contiguous()
            stride = 1
        D = torch.empty(P, 8, device=self.device)
        I = torch.empty(P, 8, dtype=torch.int32, device=self.device)
        n = torch.empty(P, dtype=torch.int32, device=self.device)
        if self._pos.shape[0] == 0:
            D.fill_(torch.finfo(torch.float32).max); I.fill_(-1); n.zero_()
            return D, I, n
        ix = self.index_struct()
        _cabi.launch_on(self.device, 'xrd_pointslam_knn_query', C.byref(ix), ptr(pos), ptr(radius),
                        stride, P, ptr(D), ptr(I), ptr(n))
        return D, I, n

    def near_pcl_samples(self, rays_o, rays_d, target_d, far, near, num):
        """xrd_pointslam_sample_near_pcl on contiguous DEVICE f32 rays [R,3], depth [R] and
        far [1] -> (z [R,num] f32, near_mask [R] uint8).  Rays with depth keep an
        uninitialised row of z and a mask of 1."""
        dev = self.device
        R = rays_o.shape[0]
        z = torch.empty(R, num, dtype=torch.float32, device=dev)
        mask = torch.empty(R, dtype=torch.uint8, device=dev)
        ix = self.index_struct()
        _cabi.launch_on(dev, 'xrd_pointslam_sample_near_pcl', C.byref(ix), ptr(rays_o),
                        ptr(rays_d), ptr(target_d), R, ptr(far), float(near),
                        float(self.radius_query), int(num), ptr(z), ptr(mask))
        return z, mask

    def sample_near_pcl(self, rays_o, rays_d, near, far, num):
        """neural_point_cloud.py:284-348: samples of rays without depth near the cloud, on the
        device.  -> (z_vals [R,num] f32, invalid_mask [R] bool: fewer than two of the 25 march
        points from near to far have a cloud point within radius_query).  `far` (a tensor
        or a number) is taken as float32, as render_batch_ray's torch.max(far) is."""
        f32 = dict(dtype=torch.float32, device=self.device)
        rays_o = rays_o.detach().to(**f32).reshape(-1, 3).contiguous()
        rays_d = rays_d.detach().to(**f32).reshape(-1, 3).contiguous()
        far = torch.as_tensor(far).detach().to(**f32).reshape(1).contiguous()
        depth = torch.zeros(rays_o.shape[0], **f32)
        z, mask = self.near_pcl_samples(rays_o, rays_d, depth, far, near, num)
        return z, mask == 0

    # ---- map update (neural_point_cloud.py:109-221) -----------------------------
    def add_neural_points(self, batch_rays_o, batch_rays_d, batch_gt_depth, batch_gt_color=None,
                          is_pts_grad=False, dynamic_radius=None, feats=None):
        """Add N_add points per pixel whose back-projection has no neighbour within the add
        radius.  `feats` = (geo, col) overrides the N(0, 0.1) init (parity tests)."""
        dev = self.device
        ro, rd, d = (batch_rays_o.to(dev).float(), batch_rays_d.to(dev).float(),
                     batch_gt_depth.to(dev).float().reshape(-1))
        keep = d > 0
        ro, rd, d = ro[keep], rd[keep], d[keep]
        if ro.shape[0] == 0:
            return 0
        pts_gt = ro + rd * d[:, None]
        mask = torch.ones(pts_gt.shape[0], dtype=torch.bool, device=dev)
        if self._pos.shape[0] > 0:
            if dynamic_radius is not None:
                rad = dynamic_radius.to(dev).float().reshape(-1)[keep]
            else:
                rad = self.radius_min if is_pts_grad else self.radius_add
            _, _, nn_gt = self.find_neighbors(pts_gt, rad)
            mask = nn_gt == 0
        t = torch.linspace(0.0, 1.0, steps=self.N_add, device=dev)
        ds = d[:, None].repeat(1, self.N_add)
        z = self.near_end_surface * ds * (1. - t) + self.far_end_surface * ds * t
        pts = (ro[:, None, :] + rd[:, None, :] * z[..., None])[mask].reshape(-1, 3)
        n_new = pts.shape[0]
        if n_new == 0:
            return 0
        self._pos = torch.cat([self._pos, pts], 0).contiguous()
        if feats is None:
            geo = torch.zeros(n_new, self.c_dim).normal_(mean=0, std=0.1).to(dev)
            col = torch.zeros(n_new, self.c_dim).normal_(mean=0, std=0.1).to(dev)
        else:
            geo, col = feats[0].to(dev), feats[1].to(dev)
        old_g = self.geo_feats.detach() if self.geo_feats is not None else torch.zeros(0, self.c_dim, device=dev)
        old_c = self.col_feats.detach() if self.col_feats is not None else torch.zeros(0, self.c_dim, device=dev)
        self.geo_feats = nn.Parameter(torch.cat([old_g, geo], 0))
        self.col_feats = nn.Parameter(torch.cat([old_c, col], 0))
        self.frustum_mask = torch.ones(self._pos.shape[0], dtype=torch.uint8, device=dev)
        self._index = None
        return int(mask.sum())
