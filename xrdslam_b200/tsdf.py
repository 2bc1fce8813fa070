"""Block-sparse TSDF volume on the device (csrc/tsdf.cu), shaped like the parts of open3d's
ScalableTSDFVolume that get_mesh_from_RGBD uses (slam/common/common.py:622-663, reference @
f0366f20): construct with voxel_length / sdf_trunc, integrate keyframes, extract a coloured
triangle mesh.  Semantics are fixed in include/xrdslam_b200.h; parity with open3d is unpinned.

``integrate`` takes a batch of keyframes at once.  The blocks the batch touches are found on
the device (one host read: their count); storage grows to the sorted union of old and new
blocks, and every voxel then applies the batch's frames in order.  Two calls give the same
volume as one call with both batches.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _cabi
from ._cabi import XrdTsdfParams, ptr

BLOCK_RES = 16
BLOCK_VOXELS = BLOCK_RES ** 3


class TSDFVolume:
    """Device TSDF volume: ``keys`` i64 [n] (sorted packed block coordinates), ``tsdf`` /
    ``weight`` f32 [n * 4096], ``color`` f32 [n * 4096, 3] on the 0..255 scale."""

    def __init__(self, voxel_length=4.0 / 512.0, sdf_trunc=0.04, depth_trunc=1000.0, stride=4,
                 device='cuda:0'):
        if not 2.0 * sdf_trunc < BLOCK_RES * voxel_length:
            raise ValueError('sdf_trunc must be below half a block edge (8 * voxel_length)')
        self.voxel_length = float(voxel_length)
        self.sdf_trunc = float(sdf_trunc)
        self.depth_trunc = float(depth_trunc)
        self.stride = int(stride)
        self.device = torch.device(device)
        _cabi.require_cuda(self.device, 'the TSDF volume')
        self.keys = torch.empty(0, dtype=torch.int64, device=self.device)
        self.tsdf = torch.empty(0, dtype=torch.float32, device=self.device)
        self.weight = torch.empty(0, dtype=torch.float32, device=self.device)
        self.color = torch.empty(0, 3, dtype=torch.float32, device=self.device)
        self._intrinsic = (1.0, 1.0, 0.0, 0.0)

    @property
    def n_blocks(self):
        return int(self.keys.numel())

    def _params(self, intrinsic):
        fx, fy, cx, cy = (float(x) for x in intrinsic)
        return XrdTsdfParams(self.voxel_length, self.sdf_trunc, self.depth_trunc, fx, fy, cx, cy,
                             self.stride)

    def allocate(self, depth, c2w, intrinsic):
        """The blocks a batch touches: keys i64 [n] (sorted) and touched-frame masks i32
        [n, ceil(K/32)] (u32 bit patterns), on the device."""
        dev = self.device
        K, H, W = depth.shape
        P = self._params(intrinsic)
        ws, nb = _cabi.workspace(
            dev, 'tsdf_alloc', K, H, W, self.stride,
            error=f'TSDF allocation: unsupported batch shape {tuple(depth.shape)}')
        cnt = torch.empty(1, dtype=torch.int32, device=dev)
        words = (K + 31) // 32
        with torch.cuda.device(dev):
            _cabi.launch_on(dev, 'xrd_tsdf_alloc_count', ptr(depth), ptr(c2w), K, H, W,
                            C.byref(P), ptr(cnt), ptr(ws), nb)
            n = int(cnt.item())
            keys = torch.empty(n, dtype=torch.int64, device=dev)
            masks = torch.empty(n, words, dtype=torch.int32, device=dev)
            if n:
                _cabi.launch_on(dev, 'xrd_tsdf_alloc_emit', K, H, W, C.byref(P), n, ptr(keys),
                                ptr(masks), ptr(ws), nb)
        return keys, masks

    def _grow(self, keys):
        """Storage for the sorted union of the current and `keys`; returns the row of every key
        of `keys` in it."""
        if self.keys.numel() == 0:
            union = keys
        else:
            union = torch.unique(torch.cat([self.keys, keys]))
        if union.numel() != self.keys.numel():
            n = union.numel()
            tsdf = torch.zeros(n, BLOCK_VOXELS, dtype=torch.float32, device=self.device)
            weight = torch.zeros_like(tsdf)
            color = torch.zeros(n, BLOCK_VOXELS, 3, dtype=torch.float32, device=self.device)
            if self.keys.numel():
                old = torch.searchsorted(union, self.keys)
                tsdf[old] = self.tsdf.view(-1, BLOCK_VOXELS)
                weight[old] = self.weight.view(-1, BLOCK_VOXELS)
                color[old] = self.color.view(-1, BLOCK_VOXELS, 3)
            self.keys, self.tsdf = union, tsdf.view(-1)
            self.weight, self.color = weight.view(-1), color.view(-1, 3)
        return torch.searchsorted(self.keys, keys)

    def integrate(self, depth, color, c2w, intrinsic, w2c=None):
        """Fuse K frames in order.  depth f32 [K,H,W] (0 = invalid), color u8 [K,H,W,3], c2w
        f32 [K,4,4] camera-to-world in open3d axes (x right, y down, z forward), intrinsic
        (fx, fy, cx, cy).  w2c defaults to inv(c2w) in float64 rounded to float32."""
        dev = self.device
        depth = depth.to(dev, torch.float32).contiguous()
        color = color.to(dev, torch.uint8).contiguous()
        K, H, W = depth.shape
        if tuple(color.shape) != (K, H, W, 3):
            raise ValueError('color must be u8 [K,H,W,3] matching depth [K,H,W]')
        c2w_h = torch.as_tensor(c2w).detach().to('cpu', torch.float32).reshape(K, 4, 4)
        if w2c is None:
            w2c = np.linalg.inv(c2w_h.numpy().astype(np.float64)).astype(np.float32)
        w2c_d = torch.as_tensor(w2c).to('cpu', torch.float32).reshape(K, 4, 4)[:, :3].contiguous()
        c2w_d = c2w_h[:, :3].contiguous().to(dev)
        w2c_d = w2c_d.to(dev)
        keys, masks = self.allocate(depth, c2w_d, intrinsic)
        self._intrinsic = tuple(float(x) for x in intrinsic)
        if keys.numel() == 0:
            return
        rows = self._grow(keys)
        all_masks = torch.zeros(self.n_blocks, masks.shape[1], dtype=torch.int32, device=dev)
        all_masks[rows] = masks
        P = self._params(intrinsic)
        _cabi.launch_on(dev, 'xrd_tsdf_integrate', ptr(self.keys), ptr(all_masks), self.n_blocks,
                        ptr(depth), ptr(color), ptr(w2c_d), K, H, W, C.byref(P), ptr(self.tsdf),
                        ptr(self.weight), ptr(self.color))

    def extract_triangle_mesh(self):
        """-> DEVICE verts f32 [V,3], faces i32 [F,3], colors f32 [V,3] in [0,1] (nominally).
        One host read: the two totals."""
        dev = self.device
        if self.n_blocks == 0:
            return (torch.empty(0, 3, device=dev), torch.empty(0, 3, dtype=torch.int32, device=dev),
                    torch.empty(0, 3, device=dev))
        ws, nb = _cabi.workspace(
            dev, 'tsdf_mc', self.n_blocks,
            error=f'TSDF volume of {self.n_blocks} blocks is too large to mesh')
        counts = torch.empty(2, dtype=torch.int32, device=dev)
        P = self._params(self._intrinsic)
        with torch.cuda.device(dev):
            _cabi.launch_on(dev, 'xrd_tsdf_mc_count', ptr(self.keys), self.n_blocks, ptr(self.tsdf),
                            ptr(self.weight), ptr(counts), ptr(ws), nb)
            V, F = counts.tolist()
            verts = torch.empty(V, 3, dtype=torch.float32, device=dev)
            colors = torch.empty(V, 3, dtype=torch.float32, device=dev)
            faces = torch.empty(F, 3, dtype=torch.int32, device=dev)
            _cabi.launch_on(dev, 'xrd_tsdf_mc_emit', ptr(self.keys), self.n_blocks, ptr(self.tsdf),
                            ptr(self.color), C.byref(P), ptr(verts), ptr(colors), ptr(faces),
                            ptr(ws), nb)
        return verts, faces, colors


def unpack_keys(keys):
    """Packed block keys (i64) -> block coordinates i64 [n,3] (any device)."""
    k = torch.as_tensor(keys)
    m = (1 << 21) - 1
    return torch.stack([(k >> 42) & m, (k >> 21) & m, k & m], -1) - (1 << 20)


def components(faces, n_verts):
    """csrc/tsdf.cu union-find: DEVICE labels i32 [n_verts], each the smallest vertex id
    connected to it through face edges."""
    dev = faces.device
    faces = faces.to(torch.int32).contiguous()
    labels = torch.empty(n_verts, dtype=torch.int32, device=dev)
    _cabi.launch_on(dev, 'xrd_tsdf_components', ptr(faces), int(faces.shape[0]), int(n_verts),
                    ptr(labels))
    return labels


def _first_of_groups(inverse, n_groups):
    """Index of the first element of every group (inverse from torch.unique)."""
    idx = torch.arange(inverse.numel(), device=inverse.device)
    first = torch.full((n_groups,), inverse.numel(), dtype=torch.int64, device=inverse.device)
    return first.scatter_reduce_(0, inverse, idx, 'amin', include_self=True)


def clean_mesh_arrays(verts, faces, colors, min_len=100):
    """clean_mesh (common.py:666-711) on DEVICE arrays, semantics in include/xrdslam_b200.h:
    weld bit-identical positions (first occurrence keeps its colour, welded vertices in order of
    first occurrence), components over the face edges, keep those with >= min_len vertices,
    order by component (smallest vertex id) then vertex id, faces by component then original
    index, drop faces that repeat a vertex and repeated vertex sets (first kept)."""
    dev = verts.device
    V = verts.shape[0]
    if V == 0 or faces.shape[0] == 0:
        return verts[:0], faces[:0].to(torch.int32), colors[:0]
    uniq, inv = torch.unique(verts.contiguous().view(torch.int32), dim=0, return_inverse=True)
    first = _first_of_groups(inv, uniq.shape[0])
    order = torch.argsort(first)
    rank = torch.empty_like(order)
    rank[order] = torch.arange(order.numel(), device=dev)
    src = first[order]                              # welded vertex -> its first original vertex
    wv, wc = verts[src], colors[src]
    wf = rank[inv][faces.long()]                    # [F,3] welded ids
    n = wv.shape[0]
    labels = components(wf, n).long()
    referenced = torch.zeros(n, dtype=torch.bool, device=dev)
    referenced[wf.reshape(-1)] = True
    size = torch.bincount(labels[referenced], minlength=n)
    keep_v = referenced & (size[labels] >= min_len)
    vid = keep_v.nonzero().squeeze(1)
    vid = vid[torch.sort(labels[vid], stable=True).indices]
    new_id = torch.full((n,), -1, dtype=torch.int64, device=dev)
    new_id[vid] = torch.arange(vid.numel(), device=dev)
    fid = keep_v[wf[:, 0]].nonzero().squeeze(1)
    fid = fid[torch.sort(labels[wf[fid, 0]], stable=True).indices]
    nf = new_id[wf[fid]]
    nf = nf[(nf[:, 0] != nf[:, 1]) & (nf[:, 1] != nf[:, 2]) & (nf[:, 0] != nf[:, 2])]
    if nf.shape[0]:
        fu, finv = torch.unique(torch.sort(nf, 1).values, dim=0, return_inverse=True)
        ffirst = _first_of_groups(finv, fu.shape[0])
        nf = nf[ffirst[finv] == torch.arange(nf.shape[0], device=dev)]
    return wv[vid], nf.to(torch.int32), wc[vid]


def o3d_poses(c2w_list):
    """Keyframe poses f32 [K,4,4] -> (c2w with columns 1 and 2 negated, inverse in float64
    rounded to float32), as common.py:641-645 converts to open3d's camera axes."""
    c2w = np.stack([np.asarray(p, dtype=np.float32).reshape(4, 4) for p in c2w_list]).copy()
    c2w[:, :3, 1] *= -1.0
    c2w[:, :3, 2] *= -1.0
    w2c = np.linalg.inv(c2w.astype(np.float64)).astype(np.float32)
    return c2w, w2c
