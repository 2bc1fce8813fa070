"""Float64 replay of the Vox-Fusion render-and-optimise step and a checker that judges any
candidate gradient against it per embedding entry, per decoder-weight element and per ray.

ORACLE / TEST INFRASTRUCTURE -- never imported by xrdslam_b200/.

The replay restates oracle/voxfusion.py ``VoxOracle.render`` (and csrc/vox.cu, which follows the
same reference code).  What the kernel decides discretely stays fp32 and is taken as input,
exactly as the kernel computes it:
  the per-ray sample voxel ids and depths and the sample counts of the march, the fp32 sample
  points xyz = o + d * depth and their trilinear coordinates p = (xyz - centre) / voxel_size + 0.5,
  the front / back / sdf masks (z < td - tr, z > td + tr in fp32), the valid-depth mask
  0.01 < td < max_dpeth, the counts n_fs, n_sdf, n_valid, the hit-ray count Rh and the batch-wide
  S of the padded-rectangle means (SURVEY Q3), and the fp32 truncation mask z < z[first] + tr of
  sdf2weights.
Everything continuous runs in float64: p around its fp32 value (value: fp32 p, derivative:
exact), the 8 corner weights, the trilerp, the 16-128-128-129 / 144-128-3 decoder, sdf2weights,
the composite and the four weighted loss terms.  Autograd gives the float64 gradients of the
embedding table, the ten decoder tensors and the rays.

``abs_bounds`` propagates the magnitude of dL/d(colour logit, sdf) through the decoder backward
with every product replaced by |a|*|b|, so A[e] bounds the sum of absolute values of the terms
fp32 adds up for entry e; |g - g64| <= tol * A is a rounding-error statement that does not depend
on how much the terms cancel.

Ambiguity: a hidden unit with |pre| < thresh * sum|terms| may take the other ReLU branch in fp32
(or TF32); ``flip_bounds`` bounds what that changes.  A ray whose first sdf sign change, or the
sign of one of whose L1 residuals (rgb per channel, depth), differs between the candidate and
float64 takes another step for that ray: it leaves the ray and entry checks.
"""
from __future__ import annotations

import numpy as np
import torch

F64 = torch.float64
DEC_KEYS = ('w0', 'b0', 'w1', 'b1', 'ws', 'bs', 'wc0', 'bc0', 'wc1', 'bc1')
WEIGHT_KEYS = tuple('d_' + k for k in DEC_KEYS)
RAY_KEYS = ('d_rays_o', 'd_rays_d')


def _f32(v):
    """A python constant as the kernel sees it (a float config field)."""
    return float(np.float32(v))


def corner_weights(p):
    """p [P,3] -> [P,8] with corner i = qx*4 + qy*2 + qz (offset_points: x slowest)."""
    out = []
    for i in range(8):
        w = 1.0
        for d, q in enumerate(((i >> 2) & 1, (i >> 1) & 1, i & 1)):
            w = w * (p[:, d] if q else 1 - p[:, d])
        out.append(w)
    return torch.stack(out, -1)


def corner_weights_absdp(p):
    """|d w_i / d p_d| -> [P,8,3]."""
    out = torch.empty(p.shape[0], 8, 3, dtype=p.dtype, device=p.device)
    for i in range(8):
        q = ((i >> 2) & 1, (i >> 1) & 1, i & 1)
        for d in range(3):
            v = 1.0
            for e in range(3):
                if e != d:
                    v = v * (p[:, e] if q[e] else 1 - p[:, e]).abs()
            out[:, i, d] = v
    return out


# ------------------------------------------------------------- inputs ---
def from_oracle(marched, R):
    """(ray_mask [R], idx [Rh,S], depth [Rh,S], count [Rh]) from VoxOracle.march."""
    _, hits, smp = marched
    idx = smp['sampled_point_voxel_idx'].long()
    return hits, idx, smp['sampled_point_depth'], (idx >= 0).sum(1)


def from_march(m, S=None):
    """The same from SparseVoxel.last_march (device tensors, scap columns, all R rays)."""
    hits = m['ray_mask'].bool()
    S = m['s_max'] if S is None else S
    return hits, m['smp_idx'][hits][:, :S].long(), m['smp_depth'][hits][:, :S], \
        m['smp_count'][hits].long()


def prepare(rays_o, rays_d, target_s, target_d, sampled, centres, vertex_idx, voxel_size=0.2,
            trunc=0.05, max_depth=10.0, pad_depth=10.0, w=(0.5, 1.0, 5000.0, 10.0), device='cpu'):
    """The discrete, fp32 part of the step on ``sampled`` = (ray_mask, idx, depth, count) of
    ``from_oracle`` / ``from_march``.  Samples k < count[r] of every hit ray are its points,
    in (hit ray, k) order; samples k >= count carry sdf 1 and depth pad_depth."""
    dev = torch.device(device)
    f32 = dict(dtype=torch.float32, device=dev)
    ray_mask, idx, depth, count = (t.to(dev) for t in sampled)
    R = ray_mask.shape[0]
    Rh, S = idx.shape
    kk = torch.arange(S, device=dev)
    vmask = kk[None, :] < count[:, None]
    assert bool((idx[vmask] >= 0).all()) and bool((idx[~vmask] < 0).all())
    z32 = torch.where(vmask, depth.to(**f32), torch.full_like(depth.to(**f32), _f32(pad_depth)))
    ro32 = rays_o.detach().to(**f32)[ray_mask]
    rd32 = rays_d.detach().to(**f32)[ray_mask]
    ray_of, k_of = torch.nonzero(vmask, as_tuple=True)
    vox = idx[ray_of, k_of]
    cen = centres.to(**f32)[vox]
    vid = vertex_idx.to(dev).long()[vox]                     # [P,8]
    zp32 = z32[ray_of, k_of]
    vs32 = torch.tensor(_f32(voxel_size), **f32)
    # csrc/vox.cu corners(): fp32 xyz = o + d * depth, p = (xyz - centre) / vs + 0.5, no fma
    xyz32 = ro32[ray_of] + rd32[ray_of] * zp32[:, None]
    p32 = (xyz32 - cen) / vs32 + 0.5
    p0 = ((ro32.double()[ray_of] + rd32.double()[ray_of] * zp32.double()[:, None]) - cen.double()
          ) / _f32(voxel_size) + 0.5
    td32 = target_d.detach().to(**f32).reshape(-1)[ray_mask]
    tr = _f32(trunc)
    tr32 = torch.tensor(tr, **f32)
    valid = (td32 > 0.01) & (td32 < _f32(max_depth))
    front = z32 < (td32 - tr32)[:, None]
    back = z32 > (td32 + tr32)[:, None]
    smask = ~front & ~back & (td32 > 0)[:, None]
    return dict(R=R, Rh=Rh, S=S, P=int(vmask.sum()), dev=dev, ray_mask=ray_mask, count=count,
                vmask=vmask, ray_of=ray_of, k_of=k_of, flat=ray_of * S + k_of, vox=vox, vid=vid,
                cen=cen, z32=z32, ro32=ro32, rd32=rd32, xyz32=xyz32, p32=p32, p0=p0, td32=td32,
                ts64=target_s.detach().to(device=dev, dtype=F64)[ray_mask], vs=_f32(voxel_size),
                tr=tr, valid=valid, front=front, back=back, smask=smask,
                n_fs=int(front.sum()), n_sdf=int(smask.sum()), n_valid=int(valid.sum()),
                w=tuple(float(v) for v in w))


def sdf_first(sdf):
    """Index of the first sign change along the padded [Rh,S] sdf (0 when there is none)."""
    return torch.argmax(((sdf[:, 1:] * sdf[:, :-1]) < 0).to(torch.int32), dim=1)


def trunc_mask(ctx, first):
    """sdf2weights' truncation mask z < z[first] + tr, in fp32 as k_composite computes it."""
    z32 = ctx['z32']
    zlim = torch.gather(z32, 1, first[:, None]) + torch.tensor(ctx['tr'], dtype=torch.float32,
                                                                 device=z32.device)
    return (z32 < zlim) & ctx['vmask']


def forward(ctx, ro, rd, emb, dec, first=None, leaf=True, per_ray_norm=False):
    """Float64 step on the fixed discrete inputs of ``prepare``: differentiable in the hit rays
    ro/rd [Rh,3], the table emb [N,16] and the 10 decoder tensors (torch layout, DEC_KEYS order).
    ``first`` freezes the first sdf sign change of every ray (from the float64 sdf when None).
    leaf: composite on a leaf copy of the per-point (colour logits, sdf), so that dL/d raw comes
    out before the decoder backward.  per_ray_norm divides the sdf / fs sums of a ray by
    Rh * count instead of Rh * S (not the kernel's semantics: the mutation tests use it)."""
    Rh, S, dev = ctx['Rh'], ctx['S'], ctx['dev']
    ray_of, vid = ctx['ray_of'], ctx['vid']
    W0, b0, W1, b1, Ws, bs, Wc0, bc0, Wc1, bc1 = dec
    zp = ctx['z32'].double()[ray_of, ctx['k_of']]
    xyz = ro[ray_of] + rd[ray_of] * zp[:, None]
    p = ctx['p32'].double() + (((xyz - ctx['cen'].double()) / ctx['vs'] + 0.5) - ctx['p0'])
    wc = corner_weights(p)                                   # [P,8]
    x = (wc[..., None] * emb[vid]).sum(1)                    # [P,16]
    pre1 = x @ W0.T + b0
    h1 = torch.relu(pre1)
    pre2 = h1 @ W1.T + b1
    h2 = torch.relu(pre2)
    so = h2 @ Ws.T + bs
    feat = so[:, 1:]
    inc = torch.cat([feat, x], -1)
    prec = inc @ Wc0.T + bc0
    c1 = torch.relu(prec)
    logit = c1 @ Wc1.T + bc1
    raw_net = torch.cat([logit, so[:, :1]], -1)              # [P,4] colour logits ++ sdf
    for t in (x, pre1, pre2, so, prec):
        if t.requires_grad:
            t.retain_grad()
    # |pre| / sum|terms| of every hidden unit (0/0 -> inf: no terms, no decision)
    with torch.no_grad():
        aW = [v.detach().abs() for v in dec]
        M_x = (wc.abs()[..., None] * emb.detach().abs()[vid]).sum(1)
        den1 = x.abs() @ aW[0].T + aW[1]
        den2 = h1.abs() @ aW[2].T + aW[3]
        denc = inc.abs() @ aW[6].T + aW[7]
        r1 = torch.nan_to_num(pre1.abs() / den1, nan=float('inf'))
        r2 = torch.nan_to_num(pre2.abs() / den2, nan=float('inf'))
        rc = torch.nan_to_num(prec.abs() / denc, nan=float('inf'))
        # forward magnitudes: what the fp32 rounding of each operand scales with
        M_h1 = (M_x @ aW[0].T + aW[1]) * (pre1 > 0)
        M_h2 = (M_h1 @ aW[2].T + aW[3]) * (pre2 > 0)
        M_so = M_h2 @ aW[4].T + aW[5]
        M_inc = torch.cat([M_so[:, 1:], M_x], -1)
        M_c1 = (M_inc @ aW[6].T + aW[7]) * (prec > 0)
    # ---- composite (sdf2weights / raw2outputs), padded [Rh,S]
    raw = raw_net.detach().requires_grad_(True) if leaf else raw_net
    flat = ctx['flat']
    sdf = torch.ones(Rh * S, dtype=F64, device=dev).index_put((flat,), raw[:, 3]).view(Rh, S)
    col_p = torch.sigmoid(raw[:, :3])
    col = torch.zeros(Rh * S, 3, dtype=F64, device=dev).index_put((flat,), col_p).view(Rh, S, 3)
    first = sdf_first(sdf.detach()) if first is None else first
    tm = trunc_mask(ctx, first)
    tr = ctx['tr']
    a = torch.sigmoid(sdf / tr) * torch.sigmoid(-sdf / tr)
    Wn = (a * tm).sum(-1, keepdim=True) + _f32(1e-8)
    wts = a * tm / Wn
    z64 = ctx['z32'].double()
    rgb = (wts[..., None] * col).sum(1)
    depth = (wts * z64).sum(-1)
    # ---- losses (get_loss_dict): L1 rgb / depth over the valid rays, padded sdf / fs means
    w = ctx['w']
    valid, front, smask = ctx['valid'], ctx['front'].double(), ctx['smask'].double()
    td64 = ctx['td32'].double()
    n = ctx['n_fs'] + ctx['n_sdf']
    fs_w, sdf_w = 1.0 - ctx['n_fs'] / n, 1.0 - ctx['n_sdf'] / n
    res_rgb = (rgb - ctx['ts64']) * valid[:, None]
    res_d = (depth - td64) * valid
    e_sdf = (z64 + sdf * tr) - td64[:, None]
    norm = float(Rh * S) if not per_ray_norm else \
        (Rh * ctx['count'].double().clamp_min(1))[:, None]
    terms = [w[0] * res_rgb.abs().sum() / (3.0 * Rh),
             w[1] * res_d.abs().sum() / ctx['n_valid'] if ctx['n_valid'] else
             torch.tensor(float('nan'), dtype=F64, device=dev),
             w[2] * sdf_w * (e_sdf ** 2 * smask / norm).sum(),
             w[3] * fs_w * ((sdf - 1.0) ** 2 * front / norm).sum()]
    total = sum(t for t in terms if not bool(torch.isnan(t.detach())))
    return dict(locals(), terms=torch.stack([t.detach() for t in terms]))


def _draw_mag(f, ctx):
    """Magnitude of dL/d(colour logit, sdf) per point with every difference replaced by the
    sum of its operands' magnitudes -> [P,4]."""
    Rh, S, tr, w = ctx['Rh'], ctx['S'], ctx['tr'], ctx['w']
    valid = ctx['valid'].double()
    with torch.no_grad():
        sdf, col, a, Wn, tm = f['sdf'], f['col'], f['a'], f['Wn'], f['tm'].double()
        z = f['z64']
        g3 = w[0] * valid / (3.0 * Rh)                                   # |d total / d rgb_c|
        gd = w[1] * valid / ctx['n_valid'] if ctx['n_valid'] else torch.zeros_like(valid)
        q = g3[:, None] * col.sum(-1) + gd[:, None] * z.abs()            # [Rh,S]
        qw = (f['wts'] * q).sum(-1, keepdim=True)
        sg = torch.sigmoid(sdf / tr)
        da = (a * (1 - 2 * sg) / tr).abs()
        ds = tm * (q + qw) / Wn * da
        fs_w = 1.0 - ctx['n_fs'] / (ctx['n_fs'] + ctx['n_sdf'])
        sdf_w = 1.0 - ctx['n_sdf'] / (ctx['n_fs'] + ctx['n_sdf'])
        RS = float(Rh * S)
        ds = ds + 2 * w[3] * fs_w / RS * (sdf.abs() + 1) * ctx['front']
        ds = ds + 2 * w[2] * sdf_w / RS * (z.abs() + sdf.abs() * tr + f['td64'].abs()[:, None]) \
            * tr * ctx['smask']
        dl = g3[:, None, None] * f['wts'][..., None] * col * (1 - col)    # [Rh,S,3]
        flat = ctx['flat']
        return torch.cat([dl.reshape(-1, 3)[flat], ds.reshape(-1)[flat, None]], -1)


def replay_step(ctx, emb, dec, first=None, per_ray_norm=False):
    """Float64 replay of one step with the table emb [N,16] and the 10 decoder tensors.
    Returns a dict of float64 tensors on the context's device."""
    dev, R, ray_mask = ctx['dev'], ctx['R'], ctx['ray_mask']
    ro = ctx['ro32'].double().requires_grad_(True)
    rd = ctx['rd32'].double().requires_grad_(True)
    emb = emb.detach().to(device=dev, dtype=F64).requires_grad_(True)
    dec = [t.detach().to(device=dev, dtype=F64).requires_grad_(True) for t in dec]
    f = forward(ctx, ro, rd, emb, dec, first=first, per_ray_norm=per_ray_norm)
    raw = f['raw']
    draw = torch.autograd.grad(f['total'], raw)[0]
    f['raw_net'].backward(draw)

    def full(g):
        out = torch.zeros(R, 3, dtype=F64, device=dev)
        out[ray_mask] = g
        return out
    g = dict(d_emb=emb.grad, d_rays_o=full(ro.grad), d_rays_d=full(rd.grad),
             **{k: t.grad for k, t in zip(WEIGHT_KEYS, dec)})
    d = lambda t: t.detach()
    return dict(
        grads=g, losses=f['terms'], ctx=ctx, emb=emb.detach(), W=[d(t) for t in dec],
        wc=d(f['wc']), absdwc=corner_weights_absdp(d(f['p'])), p=d(f['p']),
        x=d(f['x']), h1=d(f['h1']), h2=d(f['h2']), inc=d(f['inc']), c1=d(f['c1']),
        dx=f['x'].grad, dpre1=f['pre1'].grad, dpre2=f['pre2'].grad, dso=f['so'].grad,
        dprec=f['prec'].grad, draw=draw, draw_mag=_draw_mag(f, ctx),
        M_x=f['M_x'], M_h1=f['M_h1'], M_h2=f['M_h2'], M_inc=f['M_inc'], M_c1=f['M_c1'],
        m1=d(f['pre1']) > 0, m2=d(f['pre2']) > 0, mc=d(f['prec']) > 0,
        pre1_abs=d(f['pre1']).abs(), pre2_abs=d(f['pre2']).abs(), prec_abs=d(f['prec']).abs(),
        den1=f['den1'], den2=f['den2'], denc=f['denc'],
        r1=f['r1'], r2=f['r2'], rc=f['rc'], sdf=d(f['sdf']), first=f['first'],
        rgb=d(f['rgb']), depth=d(f['depth']), res_rgb=d(f['res_rgb']), res_d=d(f['res_d']))


# ------------------------------------------------------------- bounds ---
def _emb_and_rays(ref, Bx, out):
    """Scatter a per-point |dx| bound into the table bound, and carry it through the corner
    weights (d w_i / d p), 1 / voxel_size and the per-ray sums to the rays."""
    ctx = ref['ctx']
    vid = ctx['vid']
    A = torch.zeros_like(ref['emb'])
    A.index_add_(0, vid.reshape(-1), (ref['wc'].abs()[..., None] * Bx[:, None, :]).reshape(-1, 16))
    out['d_emb'] = A
    s = (ref['emb'].abs()[vid] * Bx[:, None, :]).sum(-1)                 # [P,8]
    Bp = (s[..., None] * ref['absdwc']).sum(1) / ctx['vs']               # [P,3]
    z = ctx['z32'].double()[ctx['ray_of'], ctx['k_of']].abs()
    Bo = torch.zeros(ctx['Rh'], 3, dtype=F64, device=Bx.device).index_add_(0, ctx['ray_of'], Bp)
    Bd = torch.zeros_like(Bo).index_add_(0, ctx['ray_of'], Bp * z[:, None])
    for k, v in (('d_rays_o', Bo), ('d_rays_d', Bd)):
        out[k] = torch.zeros(ctx['R'], 3, dtype=F64, device=Bx.device)
        out[k][ctx['ray_mask']] = v
    return out


def abs_bounds(ref, pmask=None):
    """Absolute-value bounds of every gradient, summed over the points where pmask [P] is true
    (all points when None).  For a subset of points every ReLU counts as open: the candidate may
    have decided them differently (a ray that takes another step)."""
    aW = [v.abs() for v in ref['W']]
    U = ref['draw_mag']
    if pmask is not None:
        U = U * pmask.double()[:, None]
    m1, m2, mc = (ref['m1'], ref['m2'], ref['mc']) if pmask is None else (True, True, True)
    Bpc = (U[:, :3] @ aW[8]) * mc
    Binc = Bpc @ aW[6]
    Bso = torch.cat([U[:, 3:], Binc[:, :128]], -1)
    Bp2 = (Bso @ aW[4]) * m2
    Bp1 = (Bp2 @ aW[2]) * m1
    Bx = Bp1 @ aW[0] + Binc[:, 128:]
    out = dict(d_w0=Bp1.T @ ref['M_x'], d_b0=Bp1.sum(0), d_w1=Bp2.T @ ref['M_h1'], d_b1=Bp2.sum(0),
               d_ws=Bso.T @ ref['M_h2'], d_bs=Bso.sum(0), d_wc0=Bpc.T @ ref['M_inc'],
               d_bc0=Bpc.sum(0), d_wc1=U[:, :3].T @ ref['M_c1'], d_bc1=U[:, :3].sum(0))
    return _emb_and_rays(ref, Bx, out)


def flip_bounds(ref, thresh):
    """How far the gradients can move when every hidden unit with |pre| < thresh * sum|terms|
    takes the other ReLU branch: the flipped unit passes or stops its float64 upstream gradient,
    its activation (at most |pre|) enters the next layer's weight gradient, and the change
    propagates downstream with |W|.  Returns (bounds, [P] bool of points with such a unit)."""
    W, aW = ref['W'], [v.abs() for v in ref['W']]
    a1, a2, ac = ref['r1'] < thresh, ref['r2'] < thresh, ref['rc'] < thresh
    # a flipped unit's activation: its |pre| plus the rounding that flipped it
    h1f = (ref['pre1_abs'] + thresh * ref['den1']) * a1
    h2f = (ref['pre2_abs'] + thresh * ref['den2']) * a2
    hcf = (ref['prec_abs'] + thresh * ref['denc']) * ac
    m1, m2, mc = ref['m1'], ref['m2'], ref['mc']
    dl = ref['draw'][:, :3]
    dpc = (dl @ W[8]).abs() * ac                              # the flipped colour units
    dinc = dpc @ aW[6]
    dso = torch.cat([torch.zeros_like(dl[:, :1]), dinc[:, :128]], -1)
    # flipped units pass (or stop) their upstream, open ones pass the change
    up2 = (ref['dso'] @ W[4]).abs() + dso @ aW[4]
    dp2 = (dso @ aW[4]) * (m2 | a2) + up2 * a2
    up1 = (ref['dpre2'] @ W[2]).abs() + dp2 @ aW[2]
    dp1 = (dp2 @ aW[2]) * (m1 | a1) + up1 * a1
    dx = dp1 @ aW[0] + dinc[:, 128:]
    out = dict(d_w0=dp1.T @ ref['M_x'], d_b0=dp1.sum(0),
               d_w1=dp2.T @ ref['M_h1'] + (ref['dpre2'].abs() + dp2).T @ h1f,
               d_b1=dp2.sum(0),
               d_ws=dso.T @ ref['M_h2'] + (ref['dso'].abs() + dso).T @ h2f,
               d_bs=dso.sum(0), d_wc0=dpc.T @ ref['M_inc'], d_bc0=dpc.sum(0),
               d_wc1=dl.abs().T @ hcf, d_bc1=torch.zeros_like(dl[0]))
    out = _emb_and_rays(ref, dx, out)
    return out, a1.any(1) | a2.any(1) | ac.any(1)


# ------------------------------------------------------------ checker ---
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


def candidate_sdf(ctx, sdf_points):
    """[Rh,S] padded sdf from a candidate's per-point sdf [P] in the replay's (ray, k) order."""
    out = torch.ones(ctx['Rh'] * ctx['S'], dtype=torch.float32, device=ctx['dev'])
    out[ctx['flat']] = sdf_points.detach().to(device=ctx['dev'], dtype=torch.float32).reshape(-1)
    return out.view(ctx['Rh'], ctx['S'])


def flip_rays(ref, cand, cand_sdf=None):
    """[Rh] bool: the candidate's first sdf sign change (cand_sdf [Rh,S], padded with 1) or the
    sign of one of its L1 residuals (cand 'rgb' [R,3], 'depth' [R]) differs from float64."""
    ctx = ref['ctx']
    dev, hm = ctx['dev'], ctx['ray_mask']
    flip = torch.zeros(ctx['Rh'], dtype=torch.bool, device=dev)
    if cand_sdf is not None:
        flip |= sdf_first(cand_sdf.to(device=dev, dtype=torch.float32)) != ref['first']
    v = ctx['valid']
    if cand.get('rgb') is not None:
        e = cand['rgb'].detach().to(device=dev, dtype=F64)[hm] - ctx['ts64']
        flip |= v & (torch.sign(e) != torch.sign(ref['res_rgb'])).any(1)
    if cand.get('depth') is not None:
        e = cand['depth'].detach().to(device=dev, dtype=F64).reshape(-1)[hm] - ctx['td32'].double()
        flip |= v & (torch.sign(e) != torch.sign(ref['res_d']))
    return flip


def compare(ref, cand, amb_thresh, cand_sdf=None):
    """Error ratios of a candidate step against the float64 replay.

    cand: {'d_emb' [N,16], 'd_dec' (10 tensors, DEC_KEYS order), 'd_rays_o', 'd_rays_d' [R,3],
    'losses' [4], 'rgb' [R,3], 'depth' [R]} (missing or None entries are not judged).
    amb_thresh: the ReLU ambiguity threshold of the candidate's arithmetic.  cand_sdf [Rh,S]:
    the candidate's own per-sample sdf (``candidate_sdf``).  Returns a report (see ``failures``)."""
    ctx = ref['ctx']
    dev, S = ctx['dev'], ctx['S']
    if 'A_all' not in ref:
        ref['A_all'] = abs_bounds(ref)
    A = ref['A_all']
    flip = flip_rays(ref, cand, cand_sdf)
    A_amb, pm = flip_bounds(ref, amb_thresh)
    fp = flip[ctx['ray_of']]
    if bool(fp.any()):
        A_fl = abs_bounds(ref, fp)   # the flip ray's whole step may differ: twice its magnitude
        A_amb = {k: v + 2 * A_fl[k] for k, v in A_amb.items()}
    pm = pm | fp
    rep = dict(n_amb_points=int(pm.sum()), n_flip_rays=int(flip.sum()))
    g64 = ref['grads']
    if cand.get('d_emb') is not None:
        g = cand['d_emb'].detach().to(device=dev, dtype=F64)
        err = (g - g64['d_emb']).abs()
        keep = torch.ones(g.shape[0], dtype=torch.bool, device=dev)
        keep[ctx['vid'][pm].reshape(-1)] = False     # rows an ambiguous point touches
        rep['entry'] = _ratio(err[keep], A['d_emb'][keep])
    dec = cand.get('d_dec')
    if dec is not None:
        for key, t in zip(WEIGHT_KEYS, dec):
            if t is not None:
                err = (_d(t, dev) - g64[key].reshape(-1)).abs()
                rep[key] = _ratio(err, A[key].reshape(-1), A_amb[key].reshape(-1))
    keep_r = torch.ones(ctx['R'], dtype=torch.bool, device=dev)
    keep_r[torch.nonzero(ctx['ray_mask']).reshape(-1)[flip]] = False
    for key in RAY_KEYS:
        if cand.get(key) is not None:
            g = cand[key].detach().to(device=dev, dtype=F64).reshape(-1, 3)
            r = g64[key]
            err = (g - r).abs()[keep_r]
            rep[key] = _ratio(err, (r.abs() + A[key])[keep_r], A_amb[key][keep_r])
    if cand.get('losses') is not None:
        lo = cand['losses'].detach().to(device=dev, dtype=F64).reshape(-1)
        r = ref['losses']
        ok = ~torch.isnan(r)
        rel = ((lo - r).abs() / r.abs().clamp_min(1e-12))[ok]
        rep['loss'] = float('inf') if bool(torch.isnan(lo[ok]).any()) else float(rel.max())
    hm = ctx['ray_mask']
    same = torch.ones(ctx['R'], dtype=torch.bool, device=dev)
    if cand_sdf is not None:   # another sign change moves the truncation window: another forward
        same[torch.nonzero(hm).reshape(-1)] = \
            sdf_first(cand_sdf.to(device=dev, dtype=torch.float32)) == ref['first']
    for key, r in (('rgb', ref['rgb']), ('depth', ref['depth'])):
        if cand.get(key) is not None:
            full = torch.zeros((ctx['R'],) + r.shape[1:], dtype=F64, device=dev)
            full[hm] = r
            e = (cand[key].detach().to(device=dev, dtype=F64).reshape(full.shape) - full).abs()
            rep['fwd_' + key] = float(e[same].max()) if bool(same.any()) else 0.0
    return rep


def failures(rep, gates):
    """Checks of a ``compare`` report that exceed their gate:
    gates = {'entry': |g-g64| / A per embedding entry, 'weight': per decoder-weight element,
    'ray': per ray and component, 'loss': rel per term, 'fwd': abs rgb and depth}."""
    out = []
    if 'entry' in rep and not rep['entry'] <= gates['entry']:
        out.append(f"entry: {rep['entry']:.3g}")
    out += [f'{k}: {rep[k]:.3g}' for k in WEIGHT_KEYS if k in rep and not rep[k] <= gates['weight']]
    out += [f'{k}: {rep[k]:.3g}' for k in RAY_KEYS if k in rep and not rep[k] <= gates['ray']]
    if 'loss' in rep and not rep['loss'] <= gates['loss']:
        out.append(f"loss: {rep['loss']:.3g}")
    out += [f'fwd_{k}: {rep["fwd_" + k]:.3g}' for k in ('rgb', 'depth')
            if 'fwd_' + k in rep and not rep['fwd_' + k] <= gates['fwd']]
    return out
