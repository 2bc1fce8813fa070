"""Float64 replay of the Point-SLAM render-and-optimise step (xrd_pointslam_step, stages
'geometry' and 'color', mapping and tracking) and a checker that judges any candidate gradient
against it per point-feature row, per colour-decoder element and per ray.

ORACLE / TEST INFRASTRUCTURE -- never imported by xrdslam_b200/.

The replay restates oracle/pointslam.py ``PointOracle.render`` / ``loss_dict`` (and
csrc/pointslam.cu, which follows the same reference code).  What the kernel defines bit for bit
stays fp32 and is an input (``prepare``), never recomputed in float64 and never under a tolerance:
  z (k_sample_z: near/far surface interpolation, the two-sided linspace of zero-depth rays),
  p = o + d * z, the squared distances ((dx^2 + dy^2) + dz^2) and r * r, and with them the
  neighbour ids (ascending (D, id), D <= r^2), the neighbour count (D < r^2), has_nb and
  valid_ray_mask.  A neighbour exactly on the radius is weighted but not counted.
Everything continuous runs in float64: p around its fp32 value (value: fp32 p, derivative exact),
the inverse-distance weights and their L1 normalisation, the 5 x 32 ReLU geometry decoder, the
per-neighbour MLP and the 5 x 128 softplus(beta = 100) colour trunk (torch's linear branch above
20 included), the occupancy compositing with its -100 fill and 1e-10 terms, the variance and both
loss forms.  Autograd gives the float64 gradients.

Discrete choices outside the bit-exact set:
  * ReLU signs of the geometry decoder: a unit with |pre| < thresh * sum|terms| may take the other
    branch in fp32.  Only that point's own backward changes, so ``compare`` exempts the geo-feature
    rows its neighbours touch and its ray, and reports the exempt shares.  A saturated sample
    (1 - alpha < SAT, reached with a steep sigmoid coefficient only) is treated the same way.
  * the signs of depth - target and colour - target, the tracking mask tmp < 10 * median (median
    element included) and the 1e3 clamp: ``decide`` evaluates them on a step's own outputs, in
    that step's precision.  ``compare`` takes the candidate's decisions (its fp32 outputs are
    themselves checked against float64), replays with them when they differ from float64's and
    counts the rays that differ (``n_flip_rays``); every ray stays checked.

Error scale: the magnitudes of dL/d occ (``_occ_bound``) and dL/d(colour logit) per sample are carried back
through both decoders, the neighbour MLP, the interpolation weights and the embeddings with every
product replaced by |a| * |b| (a softplus layer's own weight gradient also counts what rounding
its argument does to the steep derivative), so A[e] bounds the sum of absolute values of the terms fp32 adds up for
entry e and |g - g64| <= tol * A does not depend on how much the terms cancel.  An entry with
A == 0 receives no term and must be exactly 0.
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F_

F64 = torch.float64
KNN = 8
CDEC_KEYS = ('B_rel', 'nb_w1', 'nb_b1', 'nb_w2', 'nb_b2') + tuple(f'w{i}' for i in range(5)) + \
    tuple(f'b{i}' for i in range(5)) + tuple(f'wc{i}' for i in range(5)) + \
    tuple(f'bc{i}' for i in range(5)) + ('wo', 'bo')      # MLPColor.tensors() order
WEIGHT_KEYS = tuple('d_' + k for k in CDEC_KEYS)
RAY_KEYS = ('d_rays_o', 'd_rays_d')
FEAT_KEYS = ('d_geo_feats', 'd_geo_feats_exempt', 'd_col_feats')


def _f32(v):
    """A python constant as the kernel sees it (a float literal or config field)."""
    return float(np.float32(v))


TWO_PI = _f32(2 * math.pi)
EPS_D, EPS_A, EPS_T = _f32(1e-10), _f32(1e-12), _f32(1e-10)

# a sample with 1 - alpha below this has alpha == 1 within a few fp32 roundings: fp32 then passes no
# gradient where float64 still does (alpha (1 - alpha) / (1 - alpha + 1e-10)); treated as ambiguous
SAT = 1e-4

DEFAULT_CFG = dict(S=5, near_s=0.98, far_s=1.02, near_end=0.3, coef=0.1, min_nn=2, stage='color',
                   is_mapping=True, w_color=0.1, handle_dynamic=True, use_color_trk=True)


# ------------------------------------------------------------ fp32 inputs ---
def far_end(td32):
    """min(5 mean(d), max(1.2 d)) as ConvOnet2._launch computes it (on td's device)."""
    return torch.minimum(5 * td32.mean(), torch.max(td32 * 1.2)).reshape(1).float()


def sample_z32(td32, far32, S, near_s, far_s, near_end):
    """k_sample_z in fp32, one rounding per operation -> [R,S]."""
    dev = td32.device
    c = lambda v: torch.tensor(np.float32(v), device=dev)
    t = torch.linspace(0.0, 1.0, steps=S, device=dev)
    d = td32.reshape(-1, 1)
    a, b = c(near_s) * d, c(far_s) * d
    one = c(1.0)
    z_nz = a * (one - t) + b * t
    start, end = c(near_end), far32.reshape(())
    step = (end - start) / c(S - 1)
    k = torch.arange(S, device=dev)
    lo = start + step * k.float()
    hi = end - step * (S - 1 - k).float()
    z_z = torch.where(k < S // 2, lo, hi)
    return torch.where(d > 0, z_nz, z_z[None, :].expand(d.shape[0], S)).contiguous()


def _sq32(cloud, q):
    d = cloud[None, :, :] - q[:, None, :]
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def knn32(cloud, q, chunk=2048):
    """Exact 8-NN in fp32, ascending (D, id), on any device -> (D [P,8], I [P,8]; absent: FLT_MAX,
    -1).  top-9 selection, candidates ordered by (D, id); a row whose 8th and 9th distances tie
    falls back to the full stable sort."""
    N, dev = cloud.shape[0], cloud.device
    fmax = torch.finfo(torch.float32).max
    Ds, Is = [], []
    for s in range(0, q.shape[0], chunk):
        D = _sq32(cloud, q[s:s + chunk])
        if N <= KNN:
            v, i = torch.sort(D, dim=1, stable=True)
            pad = KNN - N
            v = torch.cat([v, torch.full((v.shape[0], pad), fmax, device=dev)], 1)
            i = torch.cat([i, torch.full((i.shape[0], pad), -1, device=dev, dtype=i.dtype)], 1)
        else:
            v, i = torch.topk(D, KNN + 1, dim=1, largest=False)
            o = torch.argsort(i, dim=1, stable=True)
            v, i = torch.gather(v, 1, o), torch.gather(i, 1, o)
            o = torch.argsort(v, dim=1, stable=True)
            v, i = torch.gather(v, 1, o), torch.gather(i, 1, o)
            tie = torch.nonzero(v[:, KNN] == v[:, KNN - 1]).reshape(-1)
            v, i = v[:, :KNN].clone(), i[:, :KNN].clone()
            if tie.numel():
                vs, is_ = torch.sort(D[tie], dim=1, stable=True)
                v[tie], i[tie] = vs[:, :KNN], is_[:, :KNN]
        Ds.append(v)
        Is.append(i)
    return torch.cat(Ds), torch.cat(Is)


def prepare(rays_o, rays_d, target_d, target_s, radius, cloud, fmask=None, cfg=None, far=None,
            device='cpu', radius_closed=True):
    """The discrete fp32 part of the step.  radius_closed=False drops the neighbours exactly on
    the radius (not the kernel's semantics: the mutation tests use it)."""
    dev = torch.device(device)
    c = dict(DEFAULT_CFG, **(cfg or {}))
    f32 = dict(dtype=torch.float32, device=dev)
    ro32, rd32 = rays_o.detach().to(**f32), rays_d.detach().to(**f32)
    td32 = target_d.detach().to(**f32).reshape(-1)
    R, S = ro32.shape[0], c['S']
    far32 = far_end(td32) if far is None else far.detach().to(**f32).reshape(1)
    z32 = sample_z32(td32, far32, S, c['near_s'], c['far_s'], c['near_end'])
    p32 = (ro32[:, None, :] + rd32[:, None, :] * z32[..., None]).reshape(-1, 3)
    cloud32 = cloud.detach().to(**f32)
    D32, I = knn32(cloud32, p32)
    r32 = radius.detach().to(**f32).reshape(-1)
    r2 = (r32 * r32).repeat_interleave(S)[:, None]
    inside = (D32 <= r2) if radius_closed else (D32 < r2)
    inside &= I >= 0
    I = torch.where(inside, I, torch.full_like(I, -1))
    nn = ((D32 < r2) & (I >= 0)).sum(1)
    has = nn > c['min_nn'] - 1
    valid = has.view(R, S).sum(1) >= int(S / 2 + 1)
    N = cloud32.shape[0]
    fm = torch.ones(N, dtype=torch.bool, device=dev) if fmask is None else \
        fmask.to(dev).reshape(-1).bool()
    ts = target_s if target_s is not None else torch.zeros(R, 3)
    return dict(cfg=c, R=R, S=S, P=R * S, N=N, dev=dev, ro32=ro32, rd32=rd32, td32=td32, z32=z32,
                p32=p32, p0=(ro32.double()[:, None, :] + rd32.double()[:, None, :] *
                             z32.double()[..., None]).reshape(-1, 3),
                cloud=cloud32.double(), D32=torch.where(inside, D32, torch.full_like(D32, 3.4e38)),
                I=I, nn=nn, has=has, valid=valid, nz=td32 > 0, fmask=fm, r2=r2,
                ts32=ts.detach().to(**f32), ray_of=torch.arange(R, device=dev).repeat_interleave(S))


# -------------------------------------------------------------- decisions ---
def decide(ctx, depth, unc, rgb, upper_median=False):
    """The step's discrete loss decisions on its own outputs (in their dtype; fp32 for a kernel):
    mask [R], the sign of depth - target [R] and of colour - target [R,3], and in tracking the
    unclamped rays.  Also the rays within 1e-5 (relative) of the mask or clamp threshold."""
    c = ctx['cfg']
    dt = depth.dtype
    td, ts = ctx['td32'].to(dt), ctx['ts32'].to(dt)
    depth, unc, rgb = depth.detach().reshape(-1), unc.detach().reshape(-1), rgb.detach()
    near = torch.zeros_like(ctx['nz'])
    if c['is_mapping']:
        mask = ctx['nz'] & ctx['valid'] & ~torch.isnan(depth)
        live = torch.ones_like(mask)
    else:
        eps = torch.tensor(1e-10, dtype=dt, device=depth.device)
        t = (td - depth).abs() / torch.sqrt(unc + eps)
        tmp = t if c['handle_dynamic'] else (td - depth).abs()
        srt = torch.sort(tmp).values
        med = srt[tmp.numel() // 2 if upper_median else (tmp.numel() - 1) // 2]
        lim = torch.tensor(10.0, dtype=dt, device=depth.device) * med
        mask = (tmp < lim) & ctx['nz'] & ~torch.isnan(depth) & ~torch.isnan(unc)
        live = t < 1e3
        near = ctx['nz'] & (((tmp.double() - lim.double()).abs() <= 1e-5 * lim.double()) |
                            ((t.double() - 1e3).abs() <= 1e-2))
    col_on = (c['stage'] == 'color') if c['is_mapping'] else bool(c['use_color_trk'])
    return dict(mask=mask, live=live, sd=torch.sign(depth - td), sc=torch.sign(rgb - ts),
                col_on=col_on, near=near)


def same_decisions(a, b):
    """[R] bool: rays on which two decision sets agree (signs only where they are used)."""
    m = a['mask']
    ok = (m == b['mask'])
    ok &= ~m | ((a['sd'] == b['sd']) & (a['live'] == b['live']))
    if a['col_on']:
        ok &= ~m | (a['sc'] == b['sc']).all(1)
    return ok


# ---------------------------------------------------------------- forward ---
def _softplus100(x):
    return F_.softplus(x, beta=100)


def forward(ctx, ro, rd, P, mut=None):
    """Float64 forward on the fixed discrete inputs.  P: dict(geo_feats [N,32], col_feats [N,32],
    geo=dict(B, pts_w, pts_b, fc_w, fc_b, out_w, out_b), cdec=[25 tensors, CDEC_KEYS order],
    B_col [3,20], rand_feat [32], rand_feat_color [32]).  ``mut`` names a deliberate fault (the
    mutation tests)."""
    c, dev = ctx['cfg'], ctx['dev']
    R, S, Pn = ctx['R'], ctx['S'], ctx['P']
    z = ctx['z32'].double()
    p = ctx['p32'].double() + ((ro[:, None, :] + rd[:, None, :] * z[..., None]).reshape(-1, 3)
                               - ctx['p0'])
    I = ctx['I']
    live = I >= 0
    if mut == 'dead_weighted':
        live = torch.ones_like(live)
    Ic = I.clamp_min(0)
    rel = ctx['cloud'][Ic] - p[:, None, :]                 # [P,8,3]  x - p
    D = (rel * rel).sum(-1)
    a = torch.where(live, 1.0 / (D + EPS_D), torch.zeros_like(D))
    A = a.sum(1, keepdim=True).clamp_min(EPS_A)
    w = a / (A.detach() if mut == 'no_sw' else A)
    has = ctx['has']
    keep = {}

    def k(name, t):
        if t.requires_grad:
            t.retain_grad()
        keep[name] = t
        return t
    k('D', D)
    # ---- geometry: masked features, 5 x 32 ReLU decoder
    gf = P['geo_feats']
    fm = ctx['fmask'].double()[:, None]
    nf = (gf if mut == 'geo_unmasked' else gf * fm)[Ic]
    cg = (w[..., None] * nf).sum(1)
    cg = k('cg', torch.where(has[:, None], cg, P['rand_feat'].double()[None, :].expand_as(cg)))
    g = P['geo']
    arg_g = k('arg_g', (TWO_PI * p) @ g['B'])
    e = torch.sin(arg_g)
    h = e
    ratios = []
    for l in range(5):
        pre = h @ g['pts_w'][l].T + g['pts_b'][l]
        with torch.no_grad():
            den = h.abs() @ g['pts_w'][l].abs().T + g['pts_b'][l].abs()
            ratios.append(torch.nan_to_num(pre.abs() / den, nan=float('inf')).amin(1))
            keep[f'gm{l}'] = pre.detach() > 0
        h = k(f'gh{l}', torch.relu(pre) + cg @ g['fc_w'][l].T + g['fc_b'][l])
        if l == 2:
            h = torch.cat([e, h], -1)
    occ_net = k('occ', (h @ g['out_w'].T + g['out_b']).squeeze(-1))
    fill = torch.full_like(occ_net, -100.0)
    if mut == 'no_nb_grad':
        fill = fill + (occ_net - occ_net.detach())
    occ = torch.where(has, occ_net, fill).view(R, S)
    alpha = torch.sigmoid(c_f(c['coef']) * occ)
    T = torch.cumprod(torch.cat([torch.ones(R, 1, dtype=F64, device=dev),
                                 1.0 - alpha + EPS_T], -1), -1)[:, :-1]
    wk = alpha * (T.detach() if mut == 'no_suffix' else T)
    wsum = wk.sum(-1, keepdim=True) + EPS_T
    depth_raw = (wk * z).sum(-1) / wsum.squeeze(-1)
    var = (wk * (z - depth_raw[:, None]) ** 2).sum(1)
    depth = torch.where(ctx['nz'], depth_raw, torch.zeros_like(depth_raw))
    rgb = torch.zeros(R, 3, dtype=F64, device=dev)
    col_p = torch.zeros(R, S, 3, dtype=F64, device=dev)
    if c['stage'] == 'color':
        cd = dict(zip(CDEC_KEYS, P['cdec']))
        arg_r = k('arg_r', (TWO_PI * rel) @ cd['B_rel'])   # [P,8,10]
        cf = P['col_feats']
        if mut == 'col_masked':
            cf = cf * fm
        Xn = torch.cat([torch.sin(arg_r), torch.cos(arg_r), cf[Ic]], -1)
        pre_n = k('pre_n', Xn @ cd['nb_w1'].T + cd['nb_b1'])
        Hn = k('Hn', _softplus100(pre_n))
        Fn = k('Fn', Hn @ cd['nb_w2'].T + cd['nb_b2'])
        cc = (w[..., None] * Fn).sum(1)
        cc = k('cc', torch.where(has[:, None], cc,
                                 P['rand_feat_color'].double()[None, :].expand_as(cc)))
        arg_c = k('arg_c', (TWO_PI * p) @ P['B_col'])
        ec = torch.cat([torch.sin(arg_c), torch.cos(arg_c)], -1)
        hc = ec
        for l in range(5):
            keep[f'in{l}'] = hc
            pre = k(f'pre{l}', hc @ cd[f'w{l}'].T + cd[f'b{l}'])
            hc = k(f'h{l}', _softplus100(pre) + cc @ cd[f'wc{l}'].T + cd[f'bc{l}'])
            if l == 2:
                hc = torch.cat([ec, hc], -1)
        raw = k('raw', hc @ cd['wo'].T + cd['bo'])
        keep.update(Xn=Xn, Hn=Hn, h4=hc)
        col_p = torch.sigmoid(raw).view(R, S, 3)
        rgb = (wk[..., None] * col_p).sum(-2) / wsum
    keep.update(alpha=alpha, T=T, wk=wk, wsum=wsum, col_p=col_p)
    return dict(p=p, rel=rel, w=w, live=live, z=z, depth=depth, depth_raw=depth_raw, var=var,
                rgb=rgb, keep=keep, amb_ratio=torch.stack(ratios, 1).amin(1))


def c_f(v):
    return _f32(v)


def losses(ctx, f, dec, mut=None):
    """(total with the decisions ``dec`` frozen, [geo, rgb] loss values of the step's own
    outputs)."""
    c = ctx['cfg']
    td, ts = ctx['td32'].double(), ctx['ts32'].double()
    depth, rgb = f['depth'], f['rgb']
    m = dec['mask'].double()
    wcol = c_f(c['w_color'])
    if c['is_mapping']:
        scale = torch.ones_like(depth)
        live = m
    else:
        unc = f['var'] if mut == 'unc_attached' else f['var'].detach()
        scale = 1.0 / torch.sqrt(unc + EPS_T)
        live = m * dec['live'].double()
    e = depth - td
    total = (dec['sd'].double() * e * scale * live).sum()
    val_geo = (torch.clamp(e.detach().abs() * scale.detach(), max=1e3) * m).sum()
    val_rgb = torch.zeros((), dtype=F64, device=ctx['dev'])
    if dec['col_on']:
        total = total + wcol * (dec['sc'].double() * (rgb - ts) * m[:, None]).sum()
        val_rgb = wcol * ((rgb.detach() - ts).abs() * m[:, None]).sum()
    if mut == 'zero_depth_grad':
        total = total + (f['depth_raw'] * (~ctx['nz']).double()).sum()
    return total, torch.stack([val_geo, val_rgb])


# ----------------------------------------------------------------- replay ---
def params_from_oracle(ora, rand_feat, rand_feat_color):
    """``forward``'s parameter dict from an oracle/pointslam.py PointOracle."""
    g, c = ora.geo, ora.col
    geo = dict(B=g.B, pts_w=[l.weight for l in g.pts], pts_b=[l.bias for l in g.pts],
               fc_w=[l.weight for l in g.fc_c], fc_b=[l.bias for l in g.fc_c],
               out_w=g.out.weight, out_b=g.out.bias)
    cdec = [c.B_rel, c.nb1.weight, c.nb1.bias, c.nb2.weight, c.nb2.bias] + \
        [l.weight for l in c.pts] + [l.bias for l in c.pts] + [l.weight for l in c.fc_c] + \
        [l.bias for l in c.fc_c] + [c.out.weight, c.out.bias]
    return dict(geo_feats=ora.geo_feats, col_feats=ora.col_feats, geo=geo, cdec=cdec,
                B_col=c.B, rand_feat=rand_feat, rand_feat_color=rand_feat_color)


def params_from_model(model, rand_feat, rand_feat_color):
    """The same from a ConvOnet2 (xrdslam_b200.conv_onet_pointslam)."""
    g, c = model.decoder.geo_decoder, model.decoder.color_decoder
    npc = model.neural_point_cloud
    geo = dict(B=g.embedder._B, pts_w=[l.weight for l in g.pts_linears],
               pts_b=[l.bias for l in g.pts_linears], fc_w=[l.weight for l in g.fc_c],
               fc_b=[l.bias for l in g.fc_c], out_w=g.output_linear.weight,
               out_b=g.output_linear.bias)
    return dict(geo_feats=npc.geo_feats, col_feats=npc.col_feats, geo=geo, cdec=c.tensors(),
                B_col=c.embedder._B, rand_feat=rand_feat, rand_feat_color=rand_feat_color)


def _params64(params, dev):
    t = lambda v: v.detach().to(device=dev, dtype=F64)
    P = dict(geo_feats=t(params['geo_feats']), col_feats=t(params['col_feats']),
             rand_feat=t(params['rand_feat']), rand_feat_color=t(params['rand_feat_color']),
             B_col=t(params['B_col']), cdec=[t(v) for v in params['cdec']])
    g = params['geo']
    P['geo'] = {k_: ([t(v) for v in g[k_]] if isinstance(g[k_], (list, tuple)) else t(g[k_]))
                for k_ in g}
    return P


def replay_step(ctx, params, decisions=None, mut=None):
    """Float64 replay of one step.  decisions: ``decide`` output to freeze (the step's own when
    None).  Returns float64 gradients, their error scales A, outputs and loss values."""
    dev, R, S = ctx['dev'], ctx['R'], ctx['S']
    color = ctx['cfg']['stage'] == 'color'
    P = _params64(params, dev)
    ro = ctx['ro32'].double().requires_grad_(True)
    rd = ctx['rd32'].double().requires_grad_(True)
    P['geo_feats'].requires_grad_(True)
    P['col_feats'].requires_grad_(True)
    for t in P['cdec']:
        t.requires_grad_(True)
    f = forward(ctx, ro, rd, P, mut=mut)
    own = decide(ctx, f['depth'], f['var'], f['rgb'], upper_median=(mut == 'upper_median'))
    dec = own if decisions is None else decisions
    total, vals = losses(ctx, f, dec, mut=mut)
    if total.requires_grad:
        total.backward()
    K = f['keep']
    zero = lambda t: torch.zeros_like(t)
    gr = lambda t: t.grad if (t.is_leaf or t.retains_grad) and t.grad is not None else zero(t)
    grads = dict(d_geo_feats=gr(P['geo_feats']), d_rays_o=gr(ro), d_rays_d=gr(rd))
    if color:
        grads['d_col_feats'] = gr(P['col_feats'])
        grads.update({k_: gr(t) for k_, t in zip(WEIGHT_KEYS, P['cdec'])})
    # ---- error scales: |dL/d occ| and |dL/d raw| carried back with every product as |a| * |b|
    ab = lambda name: gr(K[name]).abs()
    aK = lambda name: K[name].detach().abs()
    I, live, w = ctx['I'], f['live'], f['w'].detach()
    Ic = I.clamp_min(0)
    hasf = ctx['has'].double()[:, None]
    g = {k_: ([t.abs() for t in v] if isinstance(v, list) else v.abs()) for k_, v in P['geo'].items()}
    Bh = _occ_bound(ctx, f, dec)[:, None] * g['out_w']                     # [P,32]
    Bc, Barg = 0.0, 0.0
    for l in range(4, -1, -1):
        Bc = Bc + Bh @ g['fc_w'][l]
        Bin = (Bh * K[f'gm{l}'].double()) @ g['pts_w'][l]
        if l == 3:
            Barg, Bh = Barg + Bin[:, :93], Bin[:, 93:]
        elif l == 0:
            Barg = Barg + Bin
        else:
            Bh = Bin
    Bc = Bc * hasf
    on = (live & ctx['fmask'][Ic] & ctx['has'][:, None]).double()
    A = dict(d_geo_feats=torch.zeros(ctx['N'], 32, dtype=F64, device=dev).index_add_(
        0, Ic.reshape(-1), ((w * on)[..., None] * Bc[:, None, :]).reshape(-1, 32)))
    rel = f['rel'].detach().abs()
    nf = (P['geo_feats'].detach().abs() * ctx['fmask'].double()[:, None])[Ic]
    Bw = (nf * Bc[:, None, :]).sum(-1)                                     # |dL/dw_j|  [P,8]
    Bp = (Barg * torch.cos(K['arg_g'].detach()).abs()) @ (TWO_PI * g['B']).T
    if color:
        cd = dict(zip(CDEC_KEYS, [t.detach().abs() for t in P['cdec']]))
        fl = lambda t: t.reshape(-1, t.shape[-1])

        def cond(pre, dh, Epre):
            # |dPre| plus what the forward error of pre (Epre, in units of the rounding unit) does
            # to the steep softplus'(pre) = sigmoid(100 pre)
            sg = torch.sigmoid(100.0 * pre.detach())
            return dh * sg + dh * 100.0 * sg * (1 - sg) * Epre
        cc = aK('cc')
        Xn, Hn = aK('Xn'), aK('Hn')
        # forward error magnitudes: sin / cos of an argument a carry |a| + 1 units (a ~ 300 rad for
        # the position embedding), a layer adds the sum of its terms' magnitudes
        sgn = torch.sigmoid(100.0 * K['pre_n'].detach())
        E_Xn = torch.cat([aK('arg_r') + 1, aK('arg_r') + 1, torch.zeros_like(Xn[..., 20:])], -1)
        Epn = (E_Xn + Xn) @ cd['nb_w1'].T + cd['nb_b1']
        EFn = (sgn * Epn + 2 * Hn) @ cd['nb_w2'].T + cd['nb_b2']
        Ecc = (w[..., None] * (EFn + 2 * aK('Fn'))).sum(1) * hasf
        E_e = torch.cat([aK('arg_c') + 1, aK('arg_c') + 1], -1)
        Epre, Ein = {}, E_e
        for l in range(5):
            xin = aK(f'in{l}')
            Epre[l] = (Ein + xin) @ cd[f'w{l}'].T + cd[f'b{l}']
            Ein = torch.sigmoid(100.0 * K[f'pre{l}'].detach()) * Epre[l] + \
                (Ecc + cc) @ cd[f'wc{l}'].T + cd[f'bc{l}'] + aK(f'h{l}')
            if l == 2:
                Ein = torch.cat([E_e, Ein], -1)
        A['d_wo'], A['d_bo'] = ab('raw').T @ aK('h4'), ab('raw').sum(0)
        Bh = ab('raw') @ cd['wo']
        Bcc, Bec = 0.0, 0.0
        for l in range(4, -1, -1):
            xin = aK(f'in{l}')
            Bcc = Bcc + Bh @ cd[f'wc{l}']
            A[f'd_wc{l}'], A[f'd_bc{l}'] = Bh.T @ cc, Bh.sum(0)
            Bpre = cond(K[f'pre{l}'], Bh, Epre[l])
            A[f'd_w{l}'], A[f'd_b{l}'] = Bpre.T @ xin, Bpre.sum(0)
            Bin = (Bh * torch.sigmoid(100.0 * K[f'pre{l}'].detach())) @ cd[f'w{l}']
            if l == 3:
                Bec, Bh = Bec + Bin[:, :40], Bin[:, 40:]
            elif l == 0:
                Bec = Bec + Bin
            else:
                Bh = Bin
        Bcc = Bcc * hasf
        BFn = w[..., None] * Bcc[:, None, :]                               # [P,8,32]
        A['d_nb_w2'], A['d_nb_b2'] = fl(BFn).T @ fl(Hn), fl(BFn).sum(0)
        Bpn = cond(K['pre_n'], BFn @ cd['nb_w2'], Epn)
        A['d_nb_w1'], A['d_nb_b1'] = fl(Bpn).T @ fl(Xn), fl(Bpn).sum(0)
        BXn = ((BFn @ cd['nb_w2']) * torch.sigmoid(100.0 * K['pre_n'].detach())) @ cd['nb_w1']
        onc = (live & (w != 0) & ctx['has'][:, None]).double()[..., None]
        A['d_col_feats'] = torch.zeros(ctx['N'], 32, dtype=F64, device=dev).index_add_(
            0, Ic.reshape(-1), (BXn[..., 20:] * onc).reshape(-1, 32))
        dargb = (BXn[..., :10] * Xn[..., 10:20] + BXn[..., 10:20] * Xn[..., :10]) * onc
        A['d_B_rel'] = TWO_PI * torch.einsum('pjd,pjm->dm', rel, dargb)
        Bw = Bw + (aK('Fn') * Bcc[:, None, :]).sum(-1)
        ec = torch.cat([torch.cos(K['arg_c'].detach()), torch.sin(K['arg_c'].detach())], -1).abs()
        Bp = Bp + (Bec[:, :20] * ec[:, :20] + Bec[:, 20:] * ec[:, 20:]) @ \
            (TWO_PI * P['B_col'].abs()).T + (dargb @ (TWO_PI * cd['B_rel']).T).sum(1)
    # w = a / sum a, a = 1 / (D + eps): |dL/dD_j| <= (|dL/dw_j| + sum_i w_i |dL/dw_i|) a_j w_j
    a_j = torch.where(live, 1.0 / (K['D'].detach() + EPS_D), torch.zeros_like(w))
    BD = (Bw + (w * Bw).sum(1, keepdim=True)) * a_j * w * hasf
    Bp = Bp + (BD[..., None] * 2 * rel).sum(1)
    A['d_rays_o'] = Bp.view(R, S, 3).sum(1)
    A['d_rays_d'] = (Bp.view(R, S, 3) * f['z'].abs()[..., None]).sum(1)
    d = lambda t: t.detach()
    return dict(grads=grads, A=A, losses=vals, ctx=ctx, params=params, decisions=dec, own=own,
                depth=d(f['depth']), var=d(f['var']), rgb=d(f['rgb']), w=w, live=live,
                Bc=Bc, on_geo=w * on, amb_ratio=f['amb_ratio'], sat=(1 - K['alpha'].detach()).reshape(-1) < SAT,
                keep={k_: d(v) for k_, v in K.items()},
                dkeep={k_: d(gr(v)) for k_, v in K.items() if v.requires_grad})


def _occ_bound(ctx, f, dec):
    """|dL/d occ| per sample [P] with the differences z_k - depth and c_k - rgb of the composite's
    backward replaced by the sums of their operands' magnitudes: a ray whose weight sits on one
    sample renders depth == z_k up to rounding, and tracking multiplies that rounding by
    1 / sqrt(var)."""
    c, K = ctx['cfg'], f['keep']
    d = lambda name: K[name].detach()
    alpha, T, wk, wsum = d('alpha'), d('T'), d('wk'), d('wsum')
    m = dec['mask'].double()
    scale = torch.ones_like(m) if c['is_mapping'] else \
        dec['live'].double() / torch.sqrt(f['var'].detach() + EPS_T)
    gd = (m * scale * ctx['nz'].double())[:, None]
    E = gd * (f['z'].abs() + f['depth_raw'].detach().abs()[:, None])
    if dec['col_on'] and c['stage'] == 'color':
        gc = c_f(c['w_color']) * m[:, None, None]
        E = E + (gc * (d('col_p') + f['rgb'].detach()[:, None, :])).sum(-1)
    E = E / wsum
    after = torch.flip(torch.cumsum(torch.flip(wk * E, [1]), 1), [1]) - wk * E   # sum_{k>j} w_k E_k
    B = c_f(c['coef']) * alpha * (1 - alpha) * (T * E + after / (1 - alpha + EPS_T))
    return B.reshape(-1) * ctx['has'].double()


# ---------------------------------------------------------------- checker ---
def _ratio(err, A):
    """max err / A; an error where A == 0 (nothing may land there) or a NaN is inf."""
    err, A = err.reshape(-1), A.reshape(-1)
    if bool((torch.isnan(err) | ((A == 0) & (err > 0))).any()):
        return float('inf')
    pos = A > 0
    return float((err[pos] / A[pos]).max()) if bool(pos.any()) else 0.0


def compare(ref, cand, amb_thresh):
    """Error ratios of a candidate step against the float64 replay ``ref``.

    cand: {'d_geo_feats', 'd_col_feats' [N,32], 'd_cdec' (25 tensors, CDEC_KEYS order),
    'd_rays_o', 'd_rays_d' [R,3], 'losses' [2], 'rgb' [R,3], 'depth', 'uncertainty' [R]}; missing
    or None gradients are not judged, the three outputs are required.  Returns (report, ref used):
    the replay is redone with the candidate's loss decisions when they differ from float64's."""
    ctx = ref['ctx']
    dev = ctx['dev']
    dec = decide(ctx, cand['depth'].to(dev), cand['uncertainty'].to(dev), cand['rgb'].to(dev))
    same = same_decisions(dec, ref['own'])
    if not bool(same_decisions(dec, ref['decisions']).all()):
        ref = replay_step(ctx, ref['params'], decisions=dec)
    g64, A = ref['grads'], ref['A']
    pm = ((ref['amb_ratio'] < amb_thresh) | ref['sat']) & ctx['has']
    rep = dict(n_flip_rays=int((~same).sum()), n_near=int(dec['near'].sum()),
               amb_points=float(pm.double().mean()))
    t64 = lambda t: t.detach().to(device=dev, dtype=F64)
    if cand.get('d_geo_feats') is not None:
        keep = torch.ones(ctx['N'], dtype=torch.bool, device=dev)
        ids = ctx['I'][pm]
        keep[ids[ids >= 0]] = False
        touched = A['d_geo_feats'].amax(1) > 0
        rep['exempt_rows'] = float((~keep & touched).sum()) / max(1, int(touched.sum()))
        err = (t64(cand['d_geo_feats']) - g64['d_geo_feats']).abs()
        rep['d_geo_feats'] = _ratio(err[keep], A['d_geo_feats'][keep])
        # exempt rows: an ambiguous sample can move a row by at most twice its own share of A
        I, on = ctx['I'], ref['on_geo'] * pm.double()[:, None]
        A_amb = torch.zeros_like(A['d_geo_feats']).index_add_(
            0, I.clamp_min(0).reshape(-1), (on[..., None] * ref['Bc'][:, None, :]).reshape(-1, 32))
        rep['d_geo_feats_exempt'] = _ratio(torch.clamp(err[~keep] - 2 * A_amb[~keep], min=0.0),
                                           A['d_geo_feats'][~keep])
    if cand.get('d_col_feats') is not None and 'd_col_feats' in g64:
        rep['d_col_feats'] = _ratio((t64(cand['d_col_feats']) - g64['d_col_feats']).abs(),
                                    A['d_col_feats'])
    if cand.get('d_cdec') is not None and 'd_wo' in g64:
        for key, t in zip(WEIGHT_KEYS, cand['d_cdec']):
            rep[key] = _ratio((t64(t) - g64[key]).abs(), A[key])
    keep_r = ~pm.view(ctx['R'], ctx['S']).any(1)
    rep['exempt_rays'] = float((~keep_r).double().mean())
    for key in RAY_KEYS:
        if cand.get(key) is not None:
            err = (t64(cand[key]).reshape(-1, 3) - g64[key]).abs()
            rep[key] = _ratio(err[keep_r], A[key][keep_r])
    if cand.get('losses') is not None:
        lo, r = t64(cand['losses']).reshape(-1), ref['losses']
        rep['loss'] = float(((lo - r).abs() / r.abs().clamp_min(1.0)).max()) \
            if bool(torch.isfinite(lo).all()) else float('inf')
    for key, r in (('rgb', ref['rgb']), ('depth', ref['depth']), ('uncertainty', ref['var'])):
        e = (t64(cand[key]).reshape(r.shape) - r).abs()
        rep['fwd_' + key] = float(e.max()) if bool(torch.isfinite(e).all()) else float('inf')
    return rep, ref


def failures(rep, gates):
    """Checks of a ``compare`` report that exceed their gate: gates = {'feat': |g - g64| / A per
    feature row entry (on the rows an ambiguous sample touches: beyond twice that sample's share),
    'weight': per colour-decoder element, 'ray': per ray and component, 'loss': per term relative to max(1, |term|), 'fwd': abs rgb / depth /
    uncertainty}."""
    out = []
    for keys, gate in ((FEAT_KEYS, 'feat'), (WEIGHT_KEYS, 'weight'), (RAY_KEYS, 'ray')):
        out += [f'{k_}: {rep[k_]:.3g}' for k_ in keys if k_ in rep and not rep[k_] <= gates[gate]]
    if 'loss' in rep and not rep['loss'] <= gates['loss']:
        out.append(f"loss: {rep['loss']:.3g}")
    out += [f'{k_}: {rep[k_]:.3g}' for k_ in ('fwd_rgb', 'fwd_depth', 'fwd_uncertainty')
            if not rep[k_] <= gates['fwd']]
    return out


def worst(rep):
    """{'feat', 'weight', 'ray', 'loss', 'fwd'} -> the report's largest ratio of each kind."""
    mx = lambda keys: max([rep[k_] for k_ in keys if k_ in rep], default=0.0)
    return dict(feat=mx(FEAT_KEYS), weight=mx(WEIGHT_KEYS), ray=mx(RAY_KEYS), loss=rep.get('loss', 0.0),
                fwd=mx(('fwd_rgb', 'fwd_depth', 'fwd_uncertainty')))
