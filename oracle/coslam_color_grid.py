"""Torch restatement of Co-SLAM with a separate colour hash grid (oneGrid=False).

ORACLE / TEST INFRASTRUCTURE -- never imported by xrdslam_b200/.

The one-grid oracle (oracle/coslam.py) with the reference's second representation
(reference @ f0366f20, paths relative to the reference repository):
  slam/models/joint_encoding.py:199-234   resolution_color, embed_fn_color
  slam/model_components/encodings_coslam.py:39-53  the same HashGrid config at resolution_color
  slam/model_components/decoder_coslam.py:113-136  ColorSDFNet: colour input
                                                    [oneblob48, colour_hash32, geo15]
  slam/models/joint_encoding.py:463-481   query_color_sdf with embed_fn_color
Sampling, compositing, losses and the smoothness term (SDF grid only, :165-197) are the
one-grid oracle's.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from oracle.coslam import CoslamCfg, CoslamOracle
from oracle.tcnn_restated import HashGridRestated


class CoslamColorGridOracle(CoslamOracle):
    def __init__(self, bounding_box, cfg: CoslamCfg = None, voxel_color: float = 0.08):
        super().__init__(bounding_box, cfg)
        c = self.cfg
        dim_max = (self.bounding_box[:, 1] - self.bounding_box[:, 0]).max()
        # get_resolution (:199-210): a voxel_color above 10 is the resolution itself
        self.resolution_color = voxel_color if voxel_color > 10 else int(dim_max / voxel_color)
        pls = np.exp2(np.log2(self.resolution_color / 16) / (16 - 1))
        self.embed_fn_color = HashGridRestated(3, 16, 2, c.hashsize, 16, pls, seed=1338)
        in_col = 3 * c.pos_nbins + self.embed_fn_color.n_output_dims + c.geo_feat_dim
        self.col0 = torch.nn.Linear(in_col, c.hidden_dim_color, bias=False)

    def query_color_sdf(self, x_norm):
        embed = self.embed_fn(x_norm)
        pos = self.embedpos_fn(x_norm)
        embed_color = self.embed_fn_color(x_norm)
        h = self.sdf1(F.relu(self.sdf0(torch.cat([embed, pos], -1))))
        sdf, geo = h[..., :1], h[..., 1:]
        rgb = self.col1(F.relu(self.col0(torch.cat([pos, embed_color, geo], -1))))
        return torch.cat([rgb, sdf], -1)
