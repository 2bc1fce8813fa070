"""Torch-CPU restatement of NICE-SLAM's stratified and importance sampling (rendering_perturb > 0,
rendering_n_importance > 0) over oracle/nice.py.

ORACLE / TEST INFRASTRUCTURE -- never imported by xrdslam_b200/.

Follows (reference @ f0366f20, paths relative to the reference repository):
  slam/models/conv_onet.py:470-477   jitter of the n_samples uniform samples within their
                                     intervals, before the merge with the surface samples
  slam/models/conv_onet.py:498-520   pass 1 over the S0 samples, sample_pdf on its
                                     weights[..., 1:-1] over the float64 bin midpoints, the
                                     sorted merge and pass 2 over S0 + N samples, which alone
                                     feeds the outputs and the loss
  slam/model_components/utils.py:31-76  sample_pdf (oracle.coslam_importance.sample_pdf: the
                                     same torch calls in the same order)
The reference's call passes `device=` to sample_pdf, whose signature has no such keyword, so
the reference raises TypeError there; sample_pdf_without_device below drops the keyword -- the
only change made to the reference's behaviour -- and this restatement is pinned
bit-identically to the reference under it.

The draws are given: `noise` [R, n_samples] is the reference's torch.rand(z_vals.shape) (CPU
generator) and `u` [R, N] is sample_pdf's draw (torch.rand after it, or det_u(N) when
rendering_perturb == 0).  `z_fine` replaces the sorted merge, so that a test can run the
merged samples of another implementation through the same network.
"""
from __future__ import annotations

import contextlib

import torch

from oracle.coslam_importance import det_u, sample_pdf  # noqa: F401  (det_u re-exported)


def jitter(z_vals, noise):
    """conv_onet.py:470-477 on the uniform samples [R, n_samples] (float64)."""
    mids = .5 * (z_vals[..., 1:] + z_vals[..., :-1])
    upper = torch.cat([mids, z_vals[..., -1:]], -1)
    lower = torch.cat([z_vals[..., :1], mids], -1)
    return lower + (upper - lower) * noise


def sample_z(ora, rays_o, rays_d, gt_depth, noise=None):
    """render_batch_ray's samples (conv_onet.py:391-481) with the jitter when `noise` is given;
    gt_depth None is stage 'coarse'."""
    c = ora.cfg
    N_samples, N_surface = c.n_samples, c.n_surface
    with torch.no_grad():
        det_o = rays_o.clone().detach().unsqueeze(-1)
        det_d = rays_d.clone().detach().unsqueeze(-1)
        t = (ora.bound.unsqueeze(0) - det_o) / det_d
        far_bb, _ = torch.min(torch.max(t, dim=2)[0], dim=1)
        far_bb = far_bb.unsqueeze(-1)
        far_bb += 0.01
    t_vals = torch.linspace(0., 1., steps=N_samples)
    if gt_depth is None:
        z_vals = 0.01 * (1. - t_vals) + far_bb * t_vals
        return jitter(z_vals, noise) if noise is not None else z_vals
    gt_depth = gt_depth.reshape(-1, 1)
    near = gt_depth.repeat(1, N_samples) * 0.01
    far = torch.clamp(far_bb, 0, torch.max(gt_depth * 1.2))
    nz = gt_depth > 0
    gt_nz = gt_depth[nz].unsqueeze(-1)
    t_s = torch.linspace(0., 1., steps=N_surface).double()
    z_nz = 0.95 * gt_nz.repeat(1, N_surface) * (1. - t_s) + 1.05 * gt_nz.repeat(1, N_surface) * t_s
    z_surf = torch.zeros(gt_depth.shape[0], N_surface).double()
    nzm = nz.squeeze(-1)
    z_surf[nzm, :] = z_nz
    z_surf[~nzm, :] = 0.001 * (1. - t_s) + torch.max(gt_depth) * t_s
    z_vals = near * (1. - t_vals) + far * t_vals
    if noise is not None:
        z_vals = jitter(z_vals, noise)
    z_vals, _ = torch.sort(torch.cat([z_vals, z_surf.double()], -1), -1)
    return z_vals


def render_z(ora, rays_o, rays_d, z_vals, stage):
    """One pass of render_batch_ray over given samples: eval_points, raw2outputs_nerf_color."""
    n = rays_o.shape[0]
    pts = rays_o[..., None, :] + rays_d[..., None, :] * z_vals[..., :, None]
    raw = ora.eval_points(pts.reshape(-1, 3), stage).reshape(n, z_vals.shape[1], -1)
    rgb = raw[..., :-1]
    alpha = torch.sigmoid(10.0 * raw[..., -1])
    weights = alpha.float() * torch.cumprod(
        torch.cat([torch.ones((n, 1)), (1. - alpha + 1e-10).float()], -1).float(), -1)[:, :-1]
    rgb_map = torch.sum(weights[..., None] * rgb, -2)
    depth_map = torch.sum(weights * z_vals, -1)
    tmp = z_vals - depth_map.unsqueeze(-1)
    depth_var = torch.sum(weights * tmp * tmp, dim=1)
    return dict(rgb=rgb_map, depth=depth_map, uncertainty=depth_var, z_vals=z_vals,
                weights=weights, raw=raw)


def render(ora, rays_o, rays_d, gt_depth, stage, noise=None, u=None, z_fine=None):
    """render_batch_ray with the jitter (`noise`) and, when `u` [R, N] is given, the two
    passes.  The returned dict is pass 2's, with pass 1 under 'pass1' and the samples of
    sample_pdf under 'z_samples'."""
    z1 = sample_z(ora, rays_o, rays_d, None if stage == 'coarse' else gt_depth, noise)
    if u is None:
        return render_z(ora, rays_o, rays_d, z1, stage)
    with torch.no_grad():  # pass 1 feeds nothing but the (detached) samples
        p1 = render_z(ora, rays_o, rays_d, z1, stage)
    z_mid = .5 * (z1[..., 1:] + z1[..., :-1])
    z_samples, _, _ = sample_pdf(z_mid, p1['weights'][..., 1:-1], u)
    z_samples = z_samples.detach()
    if z_fine is None:
        z_fine, _ = torch.sort(torch.cat([z1, z_samples], -1), -1)
    out = render_z(ora, rays_o, rays_d, z_fine, stage)
    out.update(pass1=p1, z_samples=z_samples)
    return out


def step(ora, rays_o, rays_d, target_s, target_d, is_mapping, stage, noise=None, u=None,
         z_fine=None):
    """-> (outputs, loss dict, total) of one step (get_loss_dict on pass 2's outputs)."""
    out = render(ora, rays_o, rays_d, target_d, stage, noise, u, z_fine)
    ld = ora.loss_dict(out, target_s, target_d, is_mapping, stage)
    total = None
    for v in ld.values():
        total = v if total is None else total + v
    return out, ld, total


@contextlib.contextmanager
def sample_pdf_without_device():
    """Within the block, the reference's conv_onet.sample_pdf ignores the `device` keyword that
    render_batch_ray (conv_onet.py:500-504) passes and utils.py:31 does not accept.  Without it
    the reference's importance sampling raises TypeError."""
    import slam.models.conv_onet as m
    orig = m.sample_pdf

    def shim(*a, device=None, **k):
        return orig(*a, **k)
    m.sample_pdf = shim
    try:
        yield
    finally:
        m.sample_pdf = orig


# ---- gates of the device sampler against this restatement ----------------------------------
def sampler_report(zs, zs_o, inds, cdf, bins, u):
    """Per-sample offsets of candidate samples `zs` [R, N] from the restatement's `zs_o` (with its
    searchsorted `inds` and `cdf`), in widths of the bin each falls in.  A sample is `bad` when
    it is off by more than 1e-3 of its bin; the bad ones must all be explained by an ulp of the
    cdf: u within 1e-6 of a cdf value (the searchsorted index may move by one) or a cdf step
    small enough that eight float ulps of it reach 1e-3 of the bin.  `exact` is the fraction of
    samples equal bit for bit."""
    below = (inds - 1).clamp(min=0)
    above = inds.clamp(max=cdf.shape[-1] - 1)
    binw = (bins.gather(1, above) - bins.gather(1, below)).abs().clamp(min=1e-12)
    off = (zs - zs_o).abs() / binw
    near_cdf = ((u[..., None] - cdf[:, None, :]).abs() < 1e-6).any(-1)
    den = cdf.gather(1, above) - cdf.gather(1, below)
    den = torch.where(den < 1e-5, torch.ones_like(den), den)
    amplified = off <= 8 * 1.2e-7 / den
    bad = off > 1e-3
    return dict(bad=float(bad.double().mean()),
                unexplained=int((bad & ~(near_cdf | amplified)).sum()),
                exact=float((zs == zs_o).double().mean()),
                median=float(off.median()))


SAMPLER_GATES = dict(bad=2e-3, unexplained=0, exact=0.3, median=1e-6)


def sampler_failures(rep, gates=SAMPLER_GATES):
    out = [f'{k}: {rep[k]:.3g}' for k in ('bad', 'unexplained', 'median') if rep[k] > gates[k]]
    if rep['exact'] < gates['exact']:
        out.append(f"exact: {rep['exact']:.3g}")
    return out


def merged_offsets(z_cand, z_ref, z1):
    """Offsets of a candidate merge [R, S0+N] from the restatement's, element by element of the
    sorted rows, in widths of the pass-1 bin (between midpoints of z1) each reference value falls
    in.  Sorting moves no element further than the largest sample offset."""
    mids = .5 * (z1[..., 1:] + z1[..., :-1])
    i = torch.searchsorted(mids.contiguous(), z_ref.contiguous()).clamp(1, mids.shape[-1] - 1)
    binw = (mids.gather(1, i) - mids.gather(1, i - 1)).abs().clamp(min=1e-12)
    return (z_cand - z_ref).abs() / binw
