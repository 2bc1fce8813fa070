"""Torch restatement of Co-SLAM's hierarchical (importance) sampling, training_n_importance > 0.

ORACLE / TEST INFRASTRUCTURE -- never imported by xrdslam_b200/.

Follows (reference @ f0366f20, paths relative to the reference repository):
  slam/models/joint_encoding.py:296-341   coarse pass, sample_pdf, sorted merge, fine pass and
                                          the extra outputs rgb0 / disp0 / acc0 / depth0 /
                                          depth_var0 / z_std
  slam/model_components/utils.py:31-76    sample_pdf (the same torch calls, in the same order:
                                          torch.cumsum on float32 accumulates in float64 and
                                          rounds each element, which a restatement in another
                                          order would not reproduce)
  slam/models/joint_encoding.py:94-147    get_loss_dict: rgb / depth terms of both passes, sdf /
                                          fs terms of the fine pass only
It wraps either oracle (CoslamOracle, or CoslamColorGridOracle for oneGrid=False).  `u` [R,N]
is the draw of sample_pdf (torch.rand([R,N]) after the coarse pass's torch.rand(z_vals.shape),
or the linspace when det); `z_fine` replaces the sorted merge, so that a test can feed the fine
samples of another implementation through the same network.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F


def det_u(n_importance):
    """sample_pdf's det draw (utils.py:50-54)."""
    N = n_importance
    return torch.linspace(0. + 0.5 / N, 1. - 0.5 / N, steps=N)


def sample_pdf(bins, weights, u):
    """utils.py:31-76 with the uniforms `u` [R,N] given; -> (samples, inds)."""
    weights = weights + 1e-5
    pdf = weights / torch.sum(weights, -1, keepdim=True)
    cdf = torch.cumsum(pdf, -1)
    cdf = torch.cat([torch.zeros_like(cdf[..., :1]), cdf], -1)
    u = u.expand(list(cdf.shape[:-1]) + [u.shape[-1]]).contiguous()
    inds = torch.searchsorted(cdf, u, right=True)
    below = torch.max(torch.zeros_like(inds - 1), inds - 1)
    above = torch.min((cdf.shape[-1] - 1) * torch.ones_like(inds), inds)
    inds_g = torch.stack([below, above], -1)
    matched_shape = [inds_g.shape[0], inds_g.shape[1], cdf.shape[-1]]
    cdf_g = torch.gather(cdf.unsqueeze(1).expand(matched_shape), 2, inds_g)
    bins_g = torch.gather(bins.unsqueeze(1).expand(matched_shape), 2, inds_g)
    denom = (cdf_g[..., 1] - cdf_g[..., 0])
    denom = torch.where(denom < 1e-5, torch.ones_like(denom), denom)
    t = (u - cdf_g[..., 0]) / denom
    samples = bins_g[..., 0] + t * (bins_g[..., 1] - bins_g[..., 0])
    return samples, inds, cdf


def render_z(ora, rays_o, rays_d, z_vals):
    """The pass of CoslamOracle.render_rays over given z_vals [R,S] (run_network, raw2outputs)."""
    n_rays = rays_o.shape[0]
    pts = rays_o[..., None, :] + rays_d[..., None, :] * z_vals[..., :, None]
    raw = ora.query_color_sdf(ora.normalise(pts.reshape(-1, 3))).reshape(n_rays, -1, 4)
    rgb = torch.sigmoid(raw[..., :3])
    weights = ora.sdf2weights(raw[..., 3], z_vals)
    rgb_map = torch.sum(weights[..., None] * rgb, -2)
    depth_map = torch.sum(weights * z_vals, -1)
    depth_var = torch.sum(weights * torch.square(z_vals - depth_map.unsqueeze(-1)), dim=-1)
    disp_map = 1. / torch.max(1e-10 * torch.ones_like(depth_map),
                              depth_map / torch.sum(weights, -1))
    acc_map = torch.sum(weights, -1)
    return dict(rgb=rgb_map, depth=depth_map, disp_map=disp_map, acc_map=acc_map,
                depth_var=depth_var, z_vals=z_vals, raw=raw, weights=weights)


def render_rays(ora, rays_o, rays_d, target_d, noise, u, z_fine=None):
    """joint_encoding.py:250-344 with training_n_importance = u.shape[-1]; the returned dict also
    carries the coarse pass ('coarse'), z_samples, the searchsorted indices and the cdf."""
    coarse = ora.render_rays(rays_o, rays_d, target_d, noise)
    z_vals = coarse['z_vals']
    z_vals_mid = .5 * (z_vals[..., 1:] + z_vals[..., :-1])
    z_samples, inds, cdf = sample_pdf(z_vals_mid, coarse['weights'][..., 1:-1], u)
    z_samples = z_samples.detach()
    if z_fine is None:
        z_fine, _ = torch.sort(torch.cat([z_vals, z_samples], -1), -1)
    out = render_z(ora, rays_o, rays_d, z_fine)
    out.update(rgb0=coarse['rgb'], disp0=coarse['disp_map'], acc0=coarse['acc_map'],
               depth0=coarse['depth'], depth_var0=coarse['depth_var'],
               z_std=torch.std(z_samples, dim=-1, unbiased=False), coarse=coarse,
               z_samples=z_samples, inds=inds, cdf=cdf)
    return out


def loss_dict(ora, out, target_s, target_d):
    """get_loss_dict (:94-147) with the coarse outputs present: rgb and depth terms of both
    passes, each pair summed before the weight; sdf / fs of the fine pass."""
    c = ora.cfg
    ld = ora.loss_dict(out, target_s, target_d, False, True)
    valid = (target_d.squeeze(-1) > 0.) * (target_d.squeeze(-1) < c.depth_trunc)
    rgb_loss = F.mse_loss(out['rgb'], target_s) + F.mse_loss(out['rgb0'], target_s)
    depth_loss = (F.mse_loss(out['depth'][valid], target_d.squeeze(-1)[valid]) +
                  F.mse_loss(out['depth0'][valid], target_d.squeeze(-1)[valid]))
    ld['rgb_loss'] = rgb_loss * c.rgb_weight
    ld['depth_loss'] = depth_loss * c.depth_weight
    return ld


def step(ora, rays_o, rays_d, target_s, target_d, noise, u, z_fine=None):
    """-> (outputs, loss dict, total) of one training step (no smoothness term)."""
    out = render_rays(ora, rays_o, rays_d, target_d, noise, u, z_fine)
    ld = loss_dict(ora, out, target_s, target_d)
    total = None
    for v in ld.values():
        total = v if total is None else total + v
    return out, ld, total
