"""CPU restatement of Vox-Fusion's mesh-extraction queries, float64.

ORACLE / TEST INFRASTRUCTURE -- never imported by xrdslam_b200/.

Follows (reference @ f0366f20):
  slam/model_components/voxel_helpers_voxfusion.py:15-59  get_scores (lattice points
      linspace(-.5, .5, res) * voxel_size + centre, meshgrid 'ij', fp32 like the reference)
  slam/model_components/voxel_helpers_voxfusion.py:62-94  eval_points
  slam/model_components/voxel_helpers_voxfusion.py:97-166 get_features / trilinear_interp
      (the same weights as oracle/voxfusion.py VoxOracle.render), decoder VoxDecoder in float64
  slam/algorithms/voxfusion.py:205-239  the vertex -> voxel lookup: points // voxel_size
      compared with every surface voxel (O(V N)), colour 0 without a match
"""
from __future__ import annotations

import copy

import torch
import torch.nn.functional as F

from oracle.voxfusion import offset_points_q


def lattice_points(centres, voxel_size, res):
    """[B, res^3, 3] fp32 points of get_scores."""
    x = torch.linspace(-.5, .5, res)
    xx, yy, zz = torch.meshgrid(x, x, x, indexing='ij')
    s = torch.stack([xx, yy, zz], -1).float()
    s = s * voxel_size
    return s.reshape(1, -1, 3) + centres.float().unsqueeze(1)


def features(xyz, vox, centres, vertex_idx, emb, voxel_size):
    """Trilinear embedding (float64) of points xyz [P,3] inside voxels vox [P] (node ids)."""
    xyz, cen = xyz.double(), centres.double()[vox]
    feats = F.embedding(vertex_idx[vox].long(), emb.double()).view(xyz.shape[0], 8, -1)
    p = ((xyz - cen) / voxel_size + 0.5).unsqueeze(1)
    q = offset_points_q().double().unsqueeze(0)
    w = (p * q + (1 - p) * (1 - q)).prod(dim=-1, keepdim=True)
    return (w * feats).sum(1)


def decode(decoder, x):
    """VoxDecoder in float64 -> (rgb [P,3], sdf [P])."""
    dec = copy.deepcopy(decoder).double()
    with torch.no_grad():
        return dec(x)


def get_scores(decoder, vox, centres, vertex_idx, emb, voxel_size, res):
    """sdf float64 [B,res,res,res] of surface voxels vox [B] (node ids)."""
    pts = lattice_points(centres[vox], voxel_size, res)
    ids = vox[:, None].expand(-1, res ** 3).reshape(-1)
    x = features(pts.reshape(-1, 3), ids, centres, vertex_idx, emb, voxel_size)
    return decode(decoder, x)[1].reshape(-1, res, res, res)


def eval_points(decoder, xyz, vox, centres, vertex_idx, emb, voxel_size):
    """colour float64 [P,3]."""
    return decode(decoder, features(xyz, vox, centres, vertex_idx, emb, voxel_size))[0]


def vertex_voxels(verts, voxels, voxel_size):
    """voxfusion.py:205-227: index into `voxels` (surface rows [N,4]) of the voxel each vertex
    falls in (points // voxel_size == voxels[:, :3]), -1 where none does."""
    vp = torch.as_tensor(verts, dtype=torch.float32) // voxel_size
    eq = (voxels[:, :3].unsqueeze(0) == vp.unsqueeze(1)).all(-1)   # [V, N]
    nz = torch.where(eq, torch.ones_like(eq).int(), -torch.ones_like(eq).int())
    srt, idx = torch.sort(nz, dim=-1, descending=True, stable=True)
    return torch.where(srt[:, 0] != -1, idx[:, 0], torch.full_like(idx[:, 0], -1))
