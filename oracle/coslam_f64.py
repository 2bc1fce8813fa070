"""Float64 replay of the Co-SLAM step and a checker that judges any candidate gradient
against it per hash level, per table entry, per weight element and per ray.

ORACLE / TEST INFRASTRUCTURE -- never imported by xrdslam_b200/.

The replay restates oracle/coslam.py.  What the kernel decides discretely stays fp32 and is
taken as input, exactly as the kernel computes it:
  z_vals, the fp32 sample points and normalised coordinates x, the hash indices and trilinear
  weights of ``hashgrid_indices`` (pinned bit-exact against the kernel), the free-space / sdf /
  valid-depth masks and the truncation mask of sdf2weights.
Everything continuous runs in float64: the interpolation (values w, derivative dw/dx = scale as
in HashGridRestated), OneBlob, both MLPs, sdf2weights and the composite, the losses and their
normalisers.  Autograd gives the float64 gradients of the table, the four weights and the rays.

Next to every gradient the replay keeps what an absolute-value bound needs: the per-point
operands of the decoder backward.  ``abs_bounds`` propagates |dL/draw| through the decoder
backward with every product replaced by |a|*|b|, so A[e] bounds the sum of absolute values of
the terms fp32 adds up for entry e; |g - g64| <= tol * A is then a rounding-error statement that
does not depend on how much the terms cancel.

Ambiguity: a point whose hidden pre-activation satisfies |pre| < thresh * sum|terms| may take
the other ReLU branch in fp32 (or TF32).  ``ambiguity`` holds min |pre| / sum|terms| per point;
the checker picks the threshold for the candidate's arithmetic.  A ray whose first sdf sign
change falls elsewhere in the candidate's own sdf than in float64 is ambiguous as a whole.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle.tcnn_restated import hashgrid_indices

F64 = torch.float64


def _f32(v):
    """A python constant as the kernel sees it (a float config field)."""
    return float(np.float32(v))


def _quartic_cdf(u, inv_radius):
    u = u * inv_radius
    u2 = u * u
    v = (15.0 / 16.0) * u * (1 - (2.0 / 3.0) * u2 + (1.0 / 5.0) * u2 * u2) + 0.5
    return torch.clamp(v, 0.0, 1.0)


def _quartic_pdf(u, inv_radius):
    u = u * inv_radius
    u2 = u * u
    inside = (u > -1) & (u < 1)
    return torch.where(inside, (15.0 / 16.0) * (1 - u2) ** 2 * inv_radius, torch.zeros_like(u))


def oneblob64(x, nb=16):
    """OneBlobRestated in float64: x [P,3] -> [P,3*nb]."""
    edges = torch.arange(nb + 1, dtype=F64, device=x.device) / nb
    d = edges[None, None, :] - x[:, :, None]
    s = float(nb)
    cdf = _quartic_cdf(d, s) + _quartic_cdf(d - 1.0, s) + _quartic_cdf(d + 1.0, s)
    return (cdf[..., 1:] - cdf[..., :-1]).reshape(x.shape[0], 3 * nb)


def oneblob64_mag(x, nb=16):
    """Magnitude of the operands of each OneBlob bin (a difference of two CDF sums, which
    cancels in the tails): the scale of its fp32 rounding error -> [P,3*nb]."""
    edges = torch.arange(nb + 1, dtype=F64, device=x.device) / nb
    d = edges[None, None, :] - x[:, :, None]
    s = float(nb)
    cdf = _quartic_cdf(d, s) + _quartic_cdf(d - 1.0, s) + _quartic_cdf(d + 1.0, s)
    return (cdf[..., 1:] + cdf[..., :-1]).reshape(x.shape[0], 3 * nb)


def oneblob64_absdx(x, nb=16):
    """|d blob[d*nb+b] / d x_d| bounded by pdf(e_b+1 - x) + pdf(e_b - x) -> [P,3,nb]."""
    edges = torch.arange(nb + 1, dtype=F64, device=x.device) / nb
    d = edges[None, None, :] - x[:, :, None]
    s = float(nb)
    pdf = _quartic_pdf(d, s) + _quartic_pdf(d - 1.0, s) + _quartic_pdf(d + 1.0, s)
    return pdf[..., 1:] + pdf[..., :-1]


def corner_weights(w):
    """w [..., 3] -> trilinear corner weights [..., 8] (corner bit d set -> w_d)."""
    out = []
    for c in range(8):
        wc = 1.0
        for d in range(3):
            wd = w[..., d]
            wc = wc * (wd if (c >> d) & 1 else (1 - wd))
        out.append(wc)
    return torch.stack(out, -1)


def corner_weights_absdw(w):
    """|d wc / d w_d| -> [..., 8, 3]."""
    out = torch.empty(*w.shape[:-1], 8, 3, dtype=w.dtype, device=w.device)
    for c in range(8):
        for d in range(3):
            v = 1.0
            for e in range(3):
                if e != d:
                    v = v * (w[..., e] if (c >> e) & 1 else (1 - w[..., e])).abs()
            out[..., c, d] = v
    return out


def level_slices(layout):
    """[(start, stop)] of each level in the flat (entry-major, feature-minor) table."""
    F = layout['n_features']
    return [(int(o) * F, (int(o) + int(n)) * F) for o, n in zip(layout['offset'], layout['size'])]


def sdf_decision(sdf, z32, trunc32):
    """sdf2weights' discrete part on [R,S] sdf: (index of the first sign change, truncation
    mask), the mask computed in fp32 as the kernel does."""
    signs = sdf[:, 1:] * sdf[:, :-1]
    inds = torch.argmax((signs < 0).to(torch.int32), dim=1)
    z_min = torch.gather(z32, 1, inds[:, None])
    mask = z32 < (z_min + torch.tensor(trunc32, dtype=torch.float32, device=z32.device))
    return inds, mask


def prepare(ora, rays_o, rays_d, target_s, target_d, z_vals, device='cpu'):
    """The discrete, fp32 part of the step: sample points, normalised coordinates, hash
    indices and weights, as the kernel computes them."""
    lay = ora.embed_fn.table
    dev = torch.device(device)
    R, S = z_vals.shape
    f32 = dict(dtype=torch.float32, device=dev)
    ro32, rd32 = rays_o.detach().to(**f32), rays_d.detach().to(**f32)
    z32 = z_vals.detach().to(**f32)
    bb = ora.bounding_box.to(dev)
    ext = bb[:, 1] - bb[:, 0]
    # oracle/coslam.py render_rays + HashGridRestated
    pts32 = ro32[:, None, :] + rd32[:, None, :] * z32[..., None]
    x32 = ((pts32.reshape(-1, 3).double() - bb[:, 0]) / ext).float()
    idx, w32 = hashgrid_indices(x32, lay)                    # [P,L,8], [P,L,3]
    # the float64 coordinates at the fp32 rays: the carriers below are first order around them
    xn0 = (ro32.double()[:, None, :] + rd32.double()[:, None, :] * z32.double()[..., None]
           ).reshape(-1, 3).sub(bb[:, 0]).div(ext)
    return dict(cfg=ora.cfg, lay=lay, dev=dev, R=R, S=S, z32=z32, bb=bb, ext=ext, x32=x32,
                xn0=xn0, idx=idx, w32=w32, ro32=ro32, rd32=rd32,
                td32=target_d.detach().to(**f32).reshape(R, 1),
                ts64=target_s.detach().to(device=dev, dtype=F64))


def forward(ctx, ro, rd, table, Ws, loss_scale=(1., 1., 1., 1.), inds=None):
    """Float64 step on the fixed discrete inputs of ``prepare``: differentiable in the rays,
    the flat table and the four weights.  ``inds`` freezes the first sdf sign change of every
    ray (taken from the float64 sdf when None).  Returns the weighted loss terms, the total and
    the intermediates the bounds need."""
    c, lay, dev, R, S = ctx['cfg'], ctx['lay'], ctx['dev'], ctx['R'], ctx['S']
    z32, bb, ext, x32, idx, w32 = (ctx[k] for k in ('z32', 'bb', 'ext', 'x32', 'idx', 'w32'))
    td32, ts64 = ctx['td32'], ctx['ts64']
    P, L = idx.shape[0], idx.shape[1]
    W0, W1, Wc0, Wc1 = Ws
    pts = ro[:, None, :] + rd[:, None, :] * z32.double()[..., None]
    xn = (pts.reshape(-1, 3) - bb[:, 0]) / ext
    x = x32.double() + (xn - ctx['xn0'])                   # value: fp32 x, derivative: exact
    scale = torch.from_numpy(lay['scale'].astype(np.float64)).to(dev)[None, :, None]
    w = w32.double() + (x - x32.double())[:, None, :] * scale   # dw/dx = scale
    wc = corner_weights(w)                                   # [P,L,8]
    tab = table.view(-1, 2)
    feat = 0
    for k in range(8):
        feat = feat + wc[..., k, None] * tab[idx[..., k]]
    feat = feat.reshape(P, 2 * L)
    feat.retain_grad()
    blob = oneblob64(x, c.pos_nbins)
    in0 = torch.cat([feat, blob], -1)
    pre0 = in0 @ W0.T
    h0 = torch.relu(pre0)
    out1 = h0 @ W1.T
    geo = out1[:, 1:]
    inc = torch.cat([blob, geo], -1)
    prec = inc @ Wc0.T
    hc = torch.relu(prec)
    rgb_raw = hc @ Wc1.T
    raw_net = torch.cat([rgb_raw, out1[:, :1]], -1)         # [P,4] rgb logits ++ sdf
    # |pre| / sum|terms| of every hidden unit (0/0 -> inf: no terms, no decision)
    r0 = torch.nan_to_num(pre0.detach().abs() / (in0.detach().abs() @ W0.detach().abs().T),
                          nan=float('inf'))
    rc = torch.nan_to_num(prec.detach().abs() / (inc.detach().abs() @ Wc0.detach().abs().T),
                          nan=float('inf'))
    # forward magnitudes: what the fp32 rounding of each operand scales with
    aW = [v.detach().abs() for v in Ws]
    M_blob = oneblob64_mag(x.detach(), c.pos_nbins)
    M_in0 = torch.cat([(wc.detach().abs()[..., None] * table.detach().abs().view(-1, 2)[idx]
                        ).sum(2).reshape(P, 2 * L), M_blob], -1)
    M_h0 = (M_in0 @ aW[0].T) * (pre0 > 0)
    M_out1 = M_h0 @ aW[1].T
    M_inc = torch.cat([M_blob, M_out1[:, 1:]], -1)
    M_hc = (M_inc @ aW[2].T) * (prec > 0)
    # ---- composite (sdf2weights / raw2outputs) on a leaf copy of raw, so that the upstream
    # gradient dL/draw and its magnitude come out before the network backward
    raw = raw_net.detach().requires_grad_(True) if inds is None else raw_net
    raw3 = raw.reshape(R, S, 4)
    sdf = raw3[..., 3]
    M_sdf = M_out1[:, 0].reshape(R, S)
    tr = _f32(c.trunc * c.sc_factor)
    inds_, tmask = sdf_decision(sdf.detach(), z32, tr)
    if inds is not None:
        z_min = torch.gather(z32, 1, inds[:, None])
        tmask = z32 < (z_min + torch.tensor(tr, dtype=torch.float32, device=dev))
    inds = inds_ if inds is None else inds
    wts = torch.sigmoid(sdf / tr) * torch.sigmoid(-sdf / tr) * tmask.double()
    wts = wts / (wts.sum(-1, keepdim=True) + 1e-8)
    z64 = z32.double()
    rgb_map = (wts[..., None] * torch.sigmoid(raw3[..., :3])).sum(-2)
    depth = (wts * z64).sum(-1)
    # ---- losses (oracle/coslam.py loss_dict), masks and counts from fp32 comparisons
    tdv = td32.reshape(-1)
    td64 = td32.double()
    valid = (tdv > 0) & (tdv < _f32(c.depth_trunc))
    front = (z32 < (td32 - tr)).double()
    back = (z32 > (td32 + tr)).double()
    dmask = (td32 > 0).double()
    smask = (1.0 - front) * (1.0 - back) * dmask
    n_fs, n_sdf = float(front.sum()), float(smask.sum())
    n = n_fs + n_sdf
    fs_w, sdf_w = 1.0 - n_fs / n, 1.0 - n_sdf / n
    # (residual, its magnitude, weight of the mean of its squares) per loss term
    res = [(rgb_map - ts64, rgb_map.detach().abs() + ts64.abs(), c.rgb_weight),
           (depth[valid] - td64[valid, 0], depth.detach()[valid].abs() + td64[valid, 0].abs(),
            c.depth_weight),
           ((z64 + sdf * tr) * smask - td64 * smask,
            (z64.abs() + M_sdf * tr + td64.abs()) * smask, c.sdf_weight * sdf_w),
           (sdf * front - front, (M_sdf + 1.0) * front, c.fs_weight * fs_w)]
    ls = [float(v) for v in loss_scale]
    terms = torch.stack([(r ** 2).mean() * wt for r, _, wt in res])
    total = (terms * torch.tensor(ls, dtype=F64, device=dev)).sum()
    return locals()


def replay_step(ora, rays_o, rays_d, target_s, target_d, z_vals, loss_scale=(1., 1., 1., 1.),
                device='cpu'):
    """Float64 replay of one fused step with the oracle's parameters.

    rays_o/rays_d/target_s [R,3], target_d [R,1] and z_vals [R,S] are fp32 (z_vals from
    ``ora.sample_z``).  The loss is sum_k loss_scale[k] * term_k over the four weighted terms
    (rgb, depth, sdf, fs).  Returns a dict of float64 tensors on ``device``."""
    ctx = prepare(ora, rays_o, rays_d, target_s, target_d, z_vals, device)
    dev = ctx['dev']
    ro = ctx['ro32'].double().requires_grad_(True)
    rd = ctx['rd32'].double().requires_grad_(True)
    table = ora.embed_fn.params.detach().to(device=dev, dtype=F64).requires_grad_(True)
    Ws = [lin.weight.detach().to(device=dev, dtype=F64).requires_grad_(True)
          for lin in (ora.sdf0, ora.sdf1, ora.col0, ora.col1)]
    W0, W1, Wc0, Wc1 = Ws
    f = forward(ctx, ro, rd, table, Ws, loss_scale)
    c, R, S, P, L = ctx['cfg'], ctx['R'], ctx['S'], f['P'], f['L']
    total, raw, res, ls = f['total'], f['raw'], f['res'], f['ls']
    draw = torch.autograd.grad(total, raw, retain_graph=True)[0]
    # the upstream gradient with every residual replaced by its magnitude: how large the
    # rounding error of a residual can make dL/draw
    draw_mag = draw.abs()
    for k, (r, m, wt) in enumerate(res):
        if r.numel() and ls[k] != 0:
            lk = (2.0 * wt * abs(ls[k]) / r.numel()) * (m * r).sum()
            draw_mag = draw_mag + torch.autograd.grad(lk, raw, retain_graph=True)[0].abs()
    f['raw_net'].backward(draw)
    g = dict(d_table=table.grad, d_w_sdf0=W0.grad, d_w_sdf1=W1.grad, d_w_col0=Wc0.grad,
             d_w_col1=Wc1.grad, d_rays_o=ro.grad, d_rays_d=rd.grad)
    r0, rc = f['r0'], f['rc']
    return dict(
        grads=g, losses=f['terms'].detach(), R=R, S=S, layout=ctx['lay'], idx=ctx['idx'],
        wc=f['wc'].detach(), absdwc=corner_weights_absdw(f['w'].detach()),
        scale=f['scale'][0, :, 0], table=table.detach(), W=[v.detach() for v in Ws],
        M_in0=f['M_in0'], M_inc=f['M_inc'], M_h0=f['M_h0'], M_hc=f['M_hc'],
        m0=(f['pre0'] > 0).detach(), mc=(f['prec'] > 0).detach(),
        draw=draw, draw_mag=draw_mag, dfeat=f['feat'].grad.detach().reshape(P, L, 2),
        hc=f['hc'].detach(), absdblob=oneblob64_absdx(f['x'].detach(), c.pos_nbins),
        binv=1.0 / ctx['ext'], pre0_abs=f['pre0'].detach().abs(),
        prec_abs=f['prec'].detach().abs(), r0=r0, rc=rc,
        ambiguity=torch.minimum(r0.amin(1), rc.amin(1)),
        z=f['z64'], x32=ctx['x32'], sdf=f['sdf'].detach(), inds=f['inds'], trunc=f['tr'])


def _table_and_rays(ref, Bfeat, Bblob, out):
    """Scatter a per-point |dfeat| bound into the table bound, and carry |dfeat|, |dblob|
    through the corner weights and OneBlob to |dL/dx| -> pts -> rays."""
    R, S = ref['R'], ref['S']
    A_table = torch.zeros_like(ref['table']).view(-1, 2)
    contrib = ref['wc'].abs()[..., None] * Bfeat[:, :, None, :]       # [P,L,8,2]
    A_table.index_add_(0, ref['idx'].reshape(-1), contrib.reshape(-1, 2))
    out['d_table'] = A_table.reshape(-1)
    tab = ref['table'].abs().view(-1, 2)
    Bw = 0
    for f in range(2):
        tf = tab[ref['idx'], f]                                          # [P,L,8]
        Bw = Bw + (tf[..., None] * ref['absdwc']).sum(2) * Bfeat[:, :, f, None]
    Bx = (Bw * ref['scale'][None, :, None]).sum(1) + (ref['absdblob'] * Bblob).sum(-1)
    Bp = (Bx * ref['binv'][None, :]).reshape(R, S, 3)
    out['d_rays_o'] = Bp.sum(1)
    out['d_rays_d'] = (Bp * ref['z'].abs()[..., None]).sum(1)
    return out


def abs_bounds(ref, pmask=None):
    """Absolute-value bounds of every gradient, summed over the points where pmask [P] is
    true (all points when None).  For a subset of points every ReLU counts as open: the
    candidate may have decided them differently (a ray with another sdf sign change)."""
    W0, W1, Wc0, Wc1 = (v.abs() for v in ref['W'])
    U = ref['draw_mag']
    if pmask is not None:
        U = U * pmask.double()[:, None]
    P, L = ref['idx'].shape[:2]
    m0, mc = (ref['m0'], ref['mc']) if pmask is None else (True, True)
    Bprec = (U[:, :3] @ Wc1) * mc
    Binc = Bprec @ Wc0
    Bout1 = torch.cat([U[:, 3:4], Binc[:, 48:]], -1)
    Bpre0 = (Bout1 @ W1) * m0
    Bin0 = Bpre0 @ W0
    out = dict(d_w_sdf0=Bpre0.T @ ref['M_in0'], d_w_sdf1=Bout1.T @ ref['M_h0'],
               d_w_col0=Bprec.T @ ref['M_inc'], d_w_col1=U[:, :3].T @ ref['M_hc'])
    return _table_and_rays(ref, Bin0[:, :2 * L].reshape(P, L, 2),
                           (Bin0[:, 2 * L:] + Binc[:, :48]).reshape(P, 3, -1), out)


def flip_bounds(ref, thresh):
    """How far the gradients can move when every hidden unit with |pre| < thresh * sum|terms|
    takes the other ReLU branch: the flipped unit's own backward contribution, and what it
    changes downstream.  Returns (bounds, [P] bool of points with such a unit)."""
    W0, W1, Wc0, Wc1 = (v.abs() for v in ref['W'])
    a0, ac = ref['r0'] < thresh, ref['rc'] < thresh
    U = ref['draw_mag']
    P, L = ref['idx'].shape[:2]
    Bhc = U[:, :3] @ Wc1
    dprec = Bhc * ac                                         # the flipped colour units
    dinc = dprec @ Wc0
    Bout1 = torch.cat([U[:, 3:4], ((Bhc * ref['mc']) @ Wc0)[:, 48:]], -1)
    dout1 = torch.cat([torch.zeros_like(U[:, 3:4]), dinc[:, 48:]], -1)
    # sdf units: flipped ones pass (or stop) the whole upstream, open ones pass the change
    dpre0 = (dout1 @ W1) * (ref['m0'] | a0) + ((Bout1 + dout1) @ W1) * a0
    din0 = dpre0 @ W0
    out = dict(d_w_sdf0=dpre0.T @ ref['M_in0'],
               d_w_sdf1=dout1.T @ ref['M_h0'] + Bout1.T @ (ref['pre0_abs'] * a0),
               d_w_col0=dprec.T @ ref['M_inc'],
               d_w_col1=U[:, :3].T @ (ref['prec_abs'] * ac))
    out = _table_and_rays(ref, din0[:, :2 * L].reshape(P, L, 2),
                          (din0[:, 2 * L:] + dinc[:, :48]).reshape(P, 3, -1), out)
    return out, a0.any(1) | ac.any(1)


# ---------------------------------------------------------------- checker ---
WEIGHT_KEYS = ('d_w_sdf0', 'd_w_sdf1', 'd_w_col0', 'd_w_col1')
RAY_KEYS = ('d_rays_o', 'd_rays_d')


def _d(t, dev):
    return t.detach().to(device=dev, dtype=F64).reshape(-1) if t is not None else None


def _ratio(err, A, A_amb=None):
    """max of (err - A_amb)+ / A; an error where A == 0 (nothing may land there) is inf."""
    if A_amb is not None:
        err = torch.clamp(err - A_amb, min=0.0)
    bad = torch.isnan(err) | ((A == 0) & (err > 0))
    if bool(bad.any()):
        return float('inf')
    pos = A > 0
    return float((err[pos] / A[pos]).max()) if bool(pos.any()) else 0.0


def compare(ref, cand, amb_thresh, cand_sdf=None):
    """Error ratios of a candidate step against the float64 replay.

    cand: {'d_table', 'd_w_*', 'd_rays_o', 'd_rays_d', 'losses'} (missing or None entries are
    not judged).  amb_thresh: the ReLU ambiguity threshold for the candidate's arithmetic.
    cand_sdf [R,S]: the candidate's own sdf (raw[..., 3]); rays whose first sign change it puts
    elsewhere than float64 are ambiguous.  Returns a report of ratios (see ``failures``)."""
    dev = ref['sdf'].device
    R, S = ref['R'], ref['S']
    if 'A_all' not in ref:
        ref['A_all'] = abs_bounds(ref)
    A = ref['A_all']
    flip = torch.zeros(R, dtype=torch.bool, device=dev)
    if cand_sdf is not None:
        z32 = ref['z'].float()
        inds_c, _ = sdf_decision(cand_sdf.detach().to(device=dev, dtype=torch.float32)
                                 .reshape(R, S), z32, ref['trunc'])
        flip = inds_c != ref['inds']
    A_amb, pm = flip_bounds(ref, amb_thresh)
    fp = flip.repeat_interleave(S)
    if bool(fp.any()):
        A_fl = abs_bounds(ref, fp)
        A_amb = {k: v + A_fl[k] for k, v in A_amb.items()}
    pm = pm | fp
    rep = dict(n_amb_points=int(pm.sum()), n_flip_rays=int(flip.sum()))
    g64 = ref['grads']
    if cand.get('d_table') is not None:
        g, r = _d(cand['d_table'], dev), g64['d_table']
        err = (g - r).abs()
        n_ent = ref['table'].numel() // 2

        def touched_by(points):
            t = torch.zeros(n_ent, dtype=torch.bool, device=dev)
            t[ref['idx'][points].reshape(-1)] = True
            return t.repeat_interleave(2)
        # entries of ambiguous points leave the per-entry check; entries of rays with another
        # sdf sign change (a different step for that ray) leave the per-level norms too
        keep = ~touched_by(pm)
        keep_l = ~touched_by(fp)
        lv, ent = [], []
        for a, b in level_slices(ref['layout']):
            k = keep_l[a:b]
            lv.append(float((g[a:b][k] - r[a:b][k]).norm() / (r[a:b][k].norm() + 1e-300)))
            k = keep[a:b]
            ent.append(_ratio(err[a:b][k], A['d_table'][a:b][k]))
        rep['level'], rep['entry_per_level'] = lv, ent
        rep['entry'] = max(ent)
    for key in WEIGHT_KEYS:
        if cand.get(key) is not None:
            err = (_d(cand[key], dev) - g64[key].reshape(-1)).abs()
            rep[key] = _ratio(err, A[key].reshape(-1), A_amb[key].reshape(-1))
    for key in RAY_KEYS:
        if cand.get(key) is not None:
            g = cand[key].detach().to(device=dev, dtype=F64).reshape(R, 3)
            r = g64[key]
            err = (g - r).abs()[~flip]
            den = (r.abs() + A[key])[~flip]
            rep[key] = _ratio(err, den, A_amb[key][~flip])
    if cand.get('losses') is not None:
        lo = cand['losses'].detach().to(device=dev, dtype=F64).reshape(-1)
        r = ref['losses']
        ok = ~torch.isnan(r)
        rel = ((lo - r).abs() / r.abs().clamp_min(1e-12))[ok]
        rep['loss'] = float('inf') if bool(torch.isnan(lo[ok]).any()) else float(rel.max())
    return rep


def failures(rep, gates):
    """Checks of a ``compare`` report that exceed their gate:
    gates = {'level': rel L2 of each level's d_table slice, 'entry': |g-g64| / A per table
    entry, 'weight': per weight element, 'ray': per ray and component, 'loss': rel per term}."""
    out = []
    if 'level' in rep:
        out += [f'level {l}: {v:.3g}' for l, v in enumerate(rep['level']) if not v <= gates['level']]
        out += [f'entry level {l}: {v:.3g}' for l, v in enumerate(rep['entry_per_level'])
                if not v <= gates['entry']]
    out += [f'{k}: {rep[k]:.3g}' for k in WEIGHT_KEYS if k in rep and not rep[k] <= gates['weight']]
    out += [f'{k}: {rep[k]:.3g}' for k in RAY_KEYS if k in rep and not rep[k] <= gates['ray']]
    if 'loss' in rep and not rep['loss'] <= gates['loss']:
        out.append(f"loss: {rep['loss']:.3g}")
    return out


# ------------------------------------------------------------- smoothness ---
def _one_level(lay, l):
    """The layout of level l alone, its entries counted from 0."""
    out = {k: (v[l:l + 1] if isinstance(v, np.ndarray) else v) for k, v in lay.items()}
    out['offset'] = np.zeros(1, dtype=np.uint32)
    return out


def smoothness_replay(ora, smooth_rand, weight=1.0, device='cpu', sample_points=None,
                      voxel=None, margin=None, with_terms=False):
    """Float64 total-variation term of oracle/coslam.py ``smoothness`` times ``weight``, on the
    fp32 lattice coordinates and their fp32 hash indices / weights.  sample_points / voxel /
    margin default to ``ora.cfg``.  Returns (loss, d_table, A_table, layout) with A_table the
    |w_c| * |dfeat| bound (dfeat = 2 coef sum of neighbour differences, bounded by
    2 coef sum (|f| + |f_nb|)).  with_terms appends, per level, the largest number of
    (point, corner) terms that land on one table entry.

    The levels are independent (the TV term sums over feature channels), so they run one at a
    time: at 75^3 points the peak stays at a few hundred MB."""
    c = ora.cfg
    sp = c.smooth_pts if sample_points is None else int(sample_points)
    lay = ora.embed_fn.table
    dev = torch.device(device)
    x32 = ora.smooth_points(smooth_rand, sp, voxel, margin).reshape(-1, 3).float().to(dev)
    n = sp - 1
    coef = float(weight) / sp ** 3
    params = ora.embed_fn.params.detach().to(device=dev, dtype=F64)
    grad, A = torch.zeros_like(params), torch.zeros_like(params)
    loss = torch.zeros((), dtype=F64, device=dev)
    terms = []
    for l, (a, b) in enumerate(level_slices(lay)):
        idx, w32 = hashgrid_indices(x32, _one_level(lay, l))     # [P,1,8] level-local, [P,1,3]
        idx, wc = idx[:, 0], corner_weights(w32[:, 0].double())    # [P,8]
        tab = params[a:b].clone().requires_grad_(True)
        tv2 = tab.view(-1, 2)
        feat = 0
        for k in range(8):
            feat = feat + wc[:, k, None] * tv2[idx[:, k]]
        f = feat.reshape(n, n, n, 2)
        tv = sum(((torch.diff(f, dim=d)) ** 2).sum() for d in range(3))
        lv = tv * coef
        lv.backward()
        loss += lv.detach()
        grad[a:b] = tab.grad
        fa = f.detach().abs()
        B = torch.zeros_like(fa)
        for d in range(3):
            s = fa.narrow(d, 0, n - 1) + fa.narrow(d, 1, n - 1)
            B.narrow(d, 1, n - 1).add_(s)
            B.narrow(d, 0, n - 1).add_(s)
        B = (2.0 * coef * B).reshape(-1, 1, 2) * wc.abs()[..., None]
        A[a:b].view(-1, 2).index_add_(0, idx.reshape(-1), B.reshape(-1, 2))
        if with_terms:
            terms.append(int(torch.bincount(idx.reshape(-1)).max()))
        del idx, wc, feat, f, tv, lv, fa, B, tab, tv2
    out = (loss, grad, A, lay)
    return out + (terms,) if with_terms else out
