"""The float64 Point-SLAM replay (oracle/pointslam_f64.py) and its checker, on the CPU.

- The replay agrees with the fp32 oracle (oracle/pointslam.py PointOracle) at fp32 level on the
  golden fixture (mapping and tracking) and on five seeded batches (half-masked frustum, small
  radii, tracking with and without handle_dynamic, 8 samples per ray): z and valid_ray_mask bit
  for bit, outputs, loss terms and every gradient.  The fp32 CPU oracle itself stays within
  feat 2.7e-9, weight 3.1e-5, ray 4.1e-11, loss 9.4e-7 and forward 4.4e-7 of float64.
- gradcheck pins the replay's analytic gradients (rays, features, colour decoder) with the
  discrete inputs frozen.
- Mutations of the replay's own gradient that a kernel bug would produce are flagged at the gates
  test_pointslam_grad_f64_gpu.py applies to GEMM modes 0, 1 and 3, except those of
  ``NOT_SEEN`` (fault -> modes), which must stay under them (so the list cannot go stale); ``MUTATIONS`` lists
  them and ``test_mutation_floors`` prints the ratio each produces (the floors of the GPU
  file's table).

``CASES`` builds the seeded batches both files run.
"""
import numpy as np
import pytest
import torch

from helpers import load_golden_pointslam, pointslam_from_golden
from oracle import pointslam_f64 as F

# what fp32 arithmetic leaves against float64 on the CPU (worst seen: see the docstring)
FP32_GATES = dict(feat=1e-8, weight=1.2e-4, ray=1.6e-10, loss=4e-6, fwd=2e-6)


# ------------------------------------------------------------------ cases ---
def batch(R, seed, per_ray=8, noise=0.03, keep=1.0, zero_every=11, radius=(0.04, 0.06),
          origin=0.0):
    """R rays towards -z with target depths in [1.2, 1.8], a cloud of per_ray noisy points around
    every surface point (thinned to the share ``keep``), query radii radius[0] + U(0, radius[1]),
    features randn * 0.5.  origin > 0: every ray starts at its own point randn * origin (the cloud
    moves with it), so that p = o + d * z rounds in the add."""
    gen = torch.Generator().manual_seed(seed)
    rd = torch.nn.functional.normalize(
        torch.randn(R, 3, generator=gen) * torch.tensor([0.4, 0.4, 0.05]) +
        torch.tensor([0, 0, -1.0]), dim=-1)
    d = torch.rand(R, generator=gen) * 0.6 + 1.2
    ro = torch.randn(R, 3, generator=torch.Generator().manual_seed(seed + 1000)) * origin
    pos = ((ro + rd * d[:, None])[:, None, :] + torch.randn(R, per_ray, 3, generator=gen) * noise
           ).reshape(-1, 3)
    if keep < 1.0:
        pos = pos[torch.rand(pos.shape[0], generator=gen) < keep]
    N = pos.shape[0]
    td = d.clone()
    if zero_every:
        td[7::zero_every] = 0
    return dict(rays_o=ro, rays_d=rd, target_d=td,
                radius=torch.rand(R, generator=gen) * radius[1] + radius[0],
                target_s=torch.rand(R, 3, generator=gen), cloud=pos,
                geo_feats=torch.randn(N, 32, generator=gen) * 0.5,
                col_feats=torch.randn(N, 32, generator=gen) * 0.5, fmask=None, cfg={})


def _z(b, S=5):
    td = b['target_d']
    return F.sample_z32(td, F.far_end(td), S, 0.98, 1.02, 0.3)


def case_bench():        # the default mapping batch: 5000 rays x 5 samples, 40 000 points
    return batch(5000, 8)


def case_p_small():      # 8 P < 512: every GEMM of the step below the wgmma kernel's width
    return batch(12, 21, zero_every=0)


def case_p_mixed():      # P < 512 <= 8 P: trunk on mma.sync, neighbour MLP on wgmma
    return batch(100, 22)


def case_p_tail():       # P = 1535: P % 4, P % 64 and P % 128 all non-zero
    return batch(307, 23, origin=0.3)


def case_one():
    return batch(1, 24, zero_every=0)


def case_mask():         # half the cloud outside the frustum
    b = batch(600, 25, origin=0.3)
    b['fmask'] = torch.rand(b['cloud'].shape[0], generator=torch.Generator().manual_seed(1)) < 0.5
    return b


def case_sparse():       # radii of the order of the point spacing
    return batch(600, 26, noise=0.02, radius=(0.015, 0.02))


def case_on_point():     # every 5th cloud point moved onto a sample point
    b = batch(300, 27, zero_every=0)
    p = (b['rays_d'][:, None, :] * _z(b)[..., None]).reshape(-1, 3)
    ids = torch.arange(0, min(p.shape[0], b['cloud'].shape[0]), 5)
    b['cloud'][ids] = p[ids]
    return b


# trk_clamp: a ray whose whole weight sits on its middle sample renders depth == target to the
# last bit, so the sign of depth - target is a rounding matter on those rays (12 of 600 on the CPU)
FLIP_CAP_CASE = {'trk_clamp': 20}
R_EXACT = 0.0625         # r * r = 2^-8 exactly


def case_on_radius():    # cloud points at fp32 distance^2 == r * r from a sample
    b = batch(300, 28, zero_every=0)
    b['radius'][:] = R_EXACT
    p = (b['rays_d'][:, None, :] * _z(b)[..., None]).reshape(-1, 3)
    x = p.clone()
    x[:, 0] = x[:, 0] + np.float32(R_EXACT)
    ok = torch.nonzero((x[:, 0] - p[:, 0]) == R_EXACT).reshape(-1)[::7]
    b['cloud'][ok] = x[ok]
    return b


def case_shared():       # 12 points, each a neighbour of hundreds of samples
    gen = torch.Generator().manual_seed(29)
    b = batch(400, 29, zero_every=0)
    b['rays_d'] = torch.nn.functional.normalize(
        torch.randn(400, 3, generator=gen) * 0.004 + torch.tensor([0, 0, -1.0]), dim=-1)
    b['target_d'] = 1.5 + torch.randn(400, generator=gen) * 0.005
    b['cloud'] = torch.tensor([0, 0, -1.5]) + torch.randn(12, 3, generator=gen) * 0.03
    b['radius'][:] = 0.12
    b['geo_feats'], b['col_feats'] = b['geo_feats'][:12], b['col_feats'][:12]
    return b


def case_depth_edges():  # target depth 0, tiny and large between ordinary rays
    b = batch(600, 30, zero_every=0)
    b['target_d'][0:400:2] = torch.tensor([0.0, 1e-3, 60.0, 0.0]).repeat(50)
    return b


def case_depth_zero():   # every target depth 0
    b = batch(64, 31, zero_every=0)
    b['target_d'][:] = 0
    return b


def case_trk_even():     # tracking: even R, outliers beyond 10 x median
    b = batch(400, 32)
    b['target_d'][3::17] += 0.25
    b['cfg'] = dict(is_mapping=False, w_color=0.5)
    return b


def case_trk_nodyn():    # tracking with tracking_handle_dynamic off: the mask on |D - d| alone
    b = batch(600, 33)
    b['cfg'] = dict(is_mapping=False, w_color=0.5, handle_dynamic=False)
    return b


def case_trk_clamp():    # sigmoid coefficient 1: the -100 fill has alpha 0, so a ray with one
    # neighboured sample has variance 0 and t = |D - d| / 1e-5 >= 1e3; the mask on |D - d| keeps it
    b = batch(600, 33, noise=0.02, radius=(0.015, 0.02))
    b['cfg'] = dict(is_mapping=False, w_color=0.5, handle_dynamic=False, coef=1.0)
    return b


def case_trk_median():   # 2 rays: ten times the lower median excludes ray 0, the upper does not
    b = batch(2, 60, zero_every=0)
    # ray 1 has neighbours at its middle sample only, so it renders its target depth: tmp ~ 0.005
    mid = b['rays_o'][1] + b['rays_d'][1] * _z(b)[1, 2]
    b['cloud'][8:] = mid + torch.randn(8, 3, generator=torch.Generator().manual_seed(2)) * 0.002
    b['radius'][1] = 0.008
    b['cfg'] = dict(is_mapping=False, w_color=0.5)
    return b


def case_trk_nocolor():
    b = batch(300, 34)
    b['cfg'] = dict(is_mapping=False, w_color=0.5, use_color_trk=False)
    return b


def case_trk_bench():
    b = batch(5000, 8, origin=0.3)
    b['cfg'] = dict(is_mapping=False, w_color=0.5)
    return b


def case_trk_geo():      # stage 'geometry' tracking at the single-block limit of k_loss
    b = batch(8192, 35, per_ray=4)
    b['cfg'] = dict(is_mapping=False, w_color=0.5, stage='geometry')
    return b


def case_b25():          # the reference's geometry embedding scale (B std 25)
    b = batch(600, 36)
    b['geo_B_scale'] = 20.0
    return b


def _case_S(S):
    def f():
        b = batch(200, 40 + S)
        b['cfg'] = dict(S=S)
        return b
    return f


CASES = dict(bench=case_bench, p_small=case_p_small, p_mixed=case_p_mixed, p_tail=case_p_tail,
             one=case_one, S2=_case_S(2), S3=_case_S(3), S8=_case_S(8), S16=_case_S(16),
             mask=case_mask, sparse=case_sparse, on_point=case_on_point,
             on_radius=case_on_radius, shared=case_shared, depth_edges=case_depth_edges,
             depth_zero=case_depth_zero, trk_even=case_trk_even, trk_nodyn=case_trk_nodyn,
             trk_clamp=case_trk_clamp, trk_median=case_trk_median,
             trk_nocolor=case_trk_nocolor, trk_bench=case_trk_bench, trk_geo=case_trk_geo,
             b25=case_b25)


def golden_dict(b):
    """The golden fixture's decoders with the batch's cloud: pointslam_from_golden's input."""
    g = dict(load_golden_pointslam())
    g.update(cloud_pos=b['cloud'].numpy(), geo_feats=b['geo_feats'].numpy(),
             col_feats=b['col_feats'].numpy())
    if 'geo_B_scale' in b:
        g['dec.embedder._B'] = g['dec.embedder._B'] * np.float32(b['geo_B_scale'])
    return g


def case_property(name, ctx, ref=None):
    """The property the case claims, on the replay's fp32 inputs (and its float64 step)."""
    P, S, R, I, nn, has = ctx['P'], ctx['S'], ctx['R'], ctx['I'], ctx['nn'], ctx['has']
    hv = has.view(R, S)
    if name in ('bench', 'trk_bench'):
        assert R == 5000 and S == 5 and ctx['N'] == 40000
    elif name == 'p_small':
        assert 8 * ((P + 3) // 4 * 4) < 512
    elif name == 'p_mixed':
        assert P < 512 <= 8 * P
    elif name == 'p_tail':
        assert P >= 512 and P % 4 and P % 64 and P % 128
    elif name == 'one':
        assert R == 1 and bool(has.any())
    elif name in ('S2', 'S3', 'S8', 'S16'):
        assert S == int(name[1:]) and bool((~ctx['nz']).any()) and bool(ctx['valid'].any())
    elif name == 'mask':
        fm = ctx['fmask'][I.clamp_min(0)] & (I >= 0)
        both = (fm.any(1) & ((I >= 0) & ~fm).any(1) & has)
        assert 0.3 < float(ctx['fmask'].double().mean()) < 0.7 and int(both.sum()) > P // 4
    elif name == 'sparse':
        cnt = (I >= 0).sum(1)
        hist = torch.bincount(cnt, minlength=9)
        assert int(hist[2:8].sum()) > P // 4 and bool((hist[2:8] > 0).all())
        mid = ~hv[:, 1:-1] & hv[:, :-2] & hv[:, 2:]
        assert int(mid.sum()) > 5 and int((~ctx['valid']).sum()) > 5 and bool(ctx['valid'].any())
    elif name == 'on_point':
        assert int(((ctx['D32'] == 0) & (I >= 0)).sum()) > 20
    elif name == 'on_radius':
        on = (ctx['D32'] == ctx['r2']) & (I >= 0)
        assert float(ctx['r2'][0]) == R_EXACT * R_EXACT and int(on.sum()) > 20
        # weighted (kept in I) but not counted
        assert bool((nn[on.any(1)] < (I >= 0).sum(1)[on.any(1)]).all())
    elif name == 'shared':
        assert ctx['N'] == 12 and int(torch.bincount(I[I >= 0], minlength=12).min()) > 300
    elif name == 'depth_edges':
        td = ctx['td32']
        assert bool((td == 0).any()) and bool((td == 1e-3).any()) and bool((td == 60).any())
    elif name == 'depth_zero':
        assert not bool(ctx['nz'].any())
    if ref is not None and not ctx['cfg']['is_mapping']:
        dec = ref['own']
        if name == 'trk_even':
            td, d, v = ctx['td32'].double(), ref['depth'], ref['var']
            tmp = torch.sort((td - d).abs() / torch.sqrt(v + 1e-10)).values
            assert R % 2 == 0 and float(tmp[R // 2 - 1]) != float(tmp[R // 2])
            assert int((ctx['nz'] & ~dec['mask']).sum()) > 2
        if name == 'trk_clamp':
            assert int((dec['mask'] & ~dec['live']).sum()) > 20
            assert int((dec['mask'] & dec['live']).sum()) > 20
        if name == 'trk_median':
            up = F.decide(ctx, ref['depth'], ref['var'], ref['rgb'], upper_median=True)
            assert R % 2 == 0 and not torch.equal(up['mask'], dec['mask'])
        if name == 'trk_nodyn':
            assert not ctx['cfg']['handle_dynamic'] and bool(dec['mask'].any())
        if name == 'trk_geo':
            assert R == 8192 and ctx['cfg']['stage'] == 'geometry'
    if ref is not None and name == 'b25':
        assert float(ref['params']['geo']['B'].detach().std()) > 20


def build_ref(name, device='cpu', far=None):
    """(batch, ctx, params, model-side golden dict) of a case with the oracle's parameters."""
    b = CASES[name]()
    g = golden_dict(b)
    ora = pointslam_from_golden(g, 'oracle')
    ctx = F.prepare(b['rays_o'], b['rays_d'], b['target_d'], b['target_s'], b['radius'],
                    b['cloud'], b['fmask'], b['cfg'], far=far, device=device)
    rf, rfc = torch.from_numpy(g['rand_feat']), torch.from_numpy(g['rand_feat_color'])
    return b, ctx, F.params_from_oracle(ora, rf, rfc), g, ora


# -------------------------------------------------- agreement with fp32 ---
def _oracle_step(b, g, ora):
    c = dict(F.DEFAULT_CFG, **b['cfg'])
    ora.n_surface, ora.coef, ora.use_color_trk = c['S'], c['coef'], c['use_color_trk']
    ora.w_color_map = ora.w_color_trk = c['w_color']
    if b['fmask'] is not None:
        ora.frustum_mask = b['fmask'].reshape(-1, 1)
    ro, rd = b['rays_o'].clone().requires_grad_(True), b['rays_d'].clone().requires_grad_(True)
    rf, rfc = torch.from_numpy(g['rand_feat']), torch.from_numpy(g['rand_feat_color'])
    out = ora.render(ro, rd, b['target_d'], b['radius'], rf, c['stage'], rfc)
    ld = ora.loss_dict(out, b['target_d'], b['target_s'], c['is_mapping'], c['handle_dynamic'])
    sum(ld.values()).backward()
    p = F.params_from_oracle(ora, rf, rfc)
    color = c['stage'] == 'color'
    return out, dict(
        d_geo_feats=ora.geo_feats.grad, d_col_feats=ora.col_feats.grad if color else None,
        d_cdec=[t.grad for t in p['cdec']] if color else None, d_rays_o=ro.grad, d_rays_d=rd.grad,
        losses=torch.stack([ld['geo_loss'].detach(), ld.get('rgb_loss', torch.zeros(())).detach()]),
        rgb=out['rgb'].detach(), depth=out['depth'].detach(),
        uncertainty=out['uncertainty'].detach())


def _golden_case(is_mapping):
    g = load_golden_pointslam()
    t = lambda k: torch.from_numpy(g[k])
    return dict(rays_o=t('rays_o'), rays_d=t('rays_d'), target_d=t('target_d').reshape(-1),
                radius=t('radius'), target_s=t('target_s'), cloud=t('cloud_pos'),
                geo_feats=t('geo_feats'), col_feats=t('col_feats'), fmask=None,
                cfg=dict(is_mapping=is_mapping, w_color=0.1 if is_mapping else 0.5))


@pytest.mark.parametrize('which', ['golden_map', 'golden_trk', 'mask', 'sparse', 'trk_even',
                                   'trk_nodyn', 'trk_clamp', 'trk_median', 'S8'])
def test_replay_matches_fp32_oracle(which):
    b = _golden_case(which == 'golden_map') if which.startswith('golden') else CASES[which]()
    g = golden_dict(b)
    ora = pointslam_from_golden(g, 'oracle')
    out, cand = _oracle_step(b, g, ora)
    ctx = F.prepare(b['rays_o'], b['rays_d'], b['target_d'], b['target_s'], b['radius'],
                    b['cloud'], b['fmask'], b['cfg'])
    assert torch.equal(ctx['z32'], out['z_vals'])
    assert torch.equal(ctx['valid'], out['valid_ray_mask'])
    ref = F.replay_step(ctx, F.params_from_oracle(ora, torch.from_numpy(g['rand_feat']),
                                                  torch.from_numpy(g['rand_feat_color'])))
    if not which.startswith('golden'):
        case_property(which, ctx, ref)
    rep, _ = F.compare(ref, cand, 1e-5)
    assert rep['n_flip_rays'] <= FLIP_CAP_CASE.get(which, 0) and rep['n_near'] == 0
    assert rep['exempt_rows'] < 0.05 and rep['exempt_rays'] < 0.06
    gates = dict(FP32_GATES, **(dict(weight=1.0, loss=1.0) if which == 'trk_median' else {}))
    assert not F.failures(rep, gates), F.failures(rep, gates)


def test_gradcheck_replay():
    """With the discrete inputs and loss decisions frozen the replay is smooth: autograd's
    float64 gradients of the rays, of touched feature rows and of colour-decoder tensors match
    finite differences (mapping; tracking detaches the uncertainty on purpose)."""
    for is_mapping in (True,):   # tracking detaches the uncertainty: not a gradient of the loss
        b = batch(3, 50, zero_every=0)
        b['cfg'] = dict(is_mapping=is_mapping)
        g = golden_dict(b)
        ora = pointslam_from_golden(g, 'oracle')
        ctx = F.prepare(b['rays_o'], b['rays_d'], b['target_d'], b['target_s'], b['radius'],
                        b['cloud'], None, b['cfg'])
        assert bool(ctx['has'].any())
        params = F.params_from_oracle(ora, torch.from_numpy(g['rand_feat']),
                                      torch.from_numpy(g['rand_feat_color']))
        P0 = F._params64(params, 'cpu')
        dec = F.replay_step(ctx, params)['own']

        rows = torch.unique(ctx['I'][ctx['I'] >= 0])[:3]

        def total(ro, rd, gf_rows, cf_rows, b_rel, bo, b3):
            gf, cf = P0['geo_feats'].clone(), P0['col_feats'].clone()
            gf[rows], cf[rows] = gf_rows, cf_rows
            P = dict(P0, geo_feats=gf, col_feats=cf)
            cd = list(P0['cdec'])
            for key, v in (('B_rel', b_rel), ('bo', bo), ('b3', b3)):
                cd[F.CDEC_KEYS.index(key)] = v
            P['cdec'] = cd
            return F.losses(ctx, F.forward(ctx, ro, rd, P), dec)[0]
        cd = dict(zip(F.CDEC_KEYS, P0['cdec']))
        args = [ctx['ro32'].double(), ctx['rd32'].double(), P0['geo_feats'][rows],
                P0['col_feats'][rows], cd['B_rel'], cd['bo'], cd['b3']]
        args = [a.clone().requires_grad_(True) for a in args]
        assert torch.autograd.gradcheck(total, args, eps=1e-7, atol=1e-7, rtol=1e-4)


# -------------------------------------------------------------- mutations ---
def _cand_of(ref):
    g = ref['grads']
    return dict(d_geo_feats=g['d_geo_feats'].clone(), d_col_feats=g['d_col_feats'].clone(),
                d_cdec=[g[k].clone() for k in F.WEIGHT_KEYS], d_rays_o=g['d_rays_o'].clone(),
                d_rays_d=g['d_rays_d'].clone(), losses=ref['losses'].clone(), rgb=ref['rgb'],
                depth=ref['depth'], uncertainty=ref['var'])


def _remut(ref, mut=None, **prep):
    """The candidate a faulty kernel would produce: the replay redone with the fault."""
    ctx = ref['ctx']
    if prep:
        b = ref['batch']
        ctx = F.prepare(b['rays_o'], b['rays_d'], b['target_d'], b['target_s'], b['radius'],
                        b['cloud'], b['fmask'], b['cfg'], **prep)
    bad = F.replay_step(ctx, ref['params'], mut=mut)
    c = _cand_of(bad)
    # a fault in the backward leaves the forward alone
    c.update(losses=ref['losses'], rgb=ref['rgb'], depth=ref['depth'], uncertainty=ref['var'])
    return c


def _w(c, key):
    return c['d_cdec'][F.WEIGHT_KEYS.index(key)]


def m_slot_shift(ref, c):       # one neighbour slot's weight taken from slot j + 1
    ctx, w, dc = ref['ctx'], ref['w'], ref['dkeep']['cg']
    p = int(torch.nonzero(((ctx['I'] >= 0).sum(1) >= 3) & ctx['has'] &
                          (dc.abs().amax(1) > 0))[0])
    c['d_geo_feats'][ctx['I'][p, 0]] += (w[p, 1] - w[p, 0]) * dc[p]


def m_ray_no_z(ref, c):         # d_rays_d without the z factor, on one ray
    r = int(torch.nonzero(ref['A']['d_rays_o'].amax(1) > 0)[0])
    c['d_rays_d'][r] = c['d_rays_o'][r]


def m_ray_copied(ref, c):       # one ray copied from its neighbour
    live = torch.nonzero(ref['A']['d_rays_o'].amax(1) > 0).reshape(-1)
    c['d_rays_o'][live[1]] = c['d_rays_o'][live[0]]
    c['d_rays_d'][live[1]] = c['d_rays_d'][live[0]]


def m_weight_1e3(ref, c):       # the most exposed element of every decoder tensor x (1 + 1e-3)
    for key in F.WEIGHT_KEYS:
        g, A = ref['grads'][key], ref['A'][key]
        i = torch.argmax(torch.where(A > 0, g.abs() / A, torch.zeros_like(A)))
        _w(c, key).view(-1)[i] *= 1 + 1e-3


def m_tail64(ref, c):           # the last 64 columns of a weight-gradient reduction dropped
    K, dK = ref['keep'], ref['dkeep']
    for l in range(5):
        _w(c, f'd_w{l}').sub_(dK[f'pre{l}'][-64:].T @ K[f'in{l}'][-64:])
        _w(c, f'd_b{l}').sub_(dK[f'pre{l}'][-64:].sum(0))
    _w(c, 'd_nb_w1').sub_(dK['pre_n'][-64:, 7].T @ K['Xn'][-64:, 7])
    _w(c, 'd_nb_w2').sub_(dK['Fn'][-64:, 7].T @ K['Hn'][-64:, 7])


def m_pad_leak(ref, c):         # three stale pad columns in the neighbour weight gradients
    K, dK = ref['keep'], ref['dkeep']
    _w(c, 'd_nb_w1').add_(dK['pre_n'][:3, 0].T @ K['Xn'][-3:, 0])
    _w(c, 'd_nb_w2').add_(dK['Fn'][:3, 0].T @ K['Hn'][-3:, 0])


# name -> (case, fault); a str fault reruns the replay with forward(mut=...)
MUTATIONS = dict(
    slot_shift=('mask', m_slot_shift), geo_unmasked=('mask', 'geo_unmasked'),
    col_masked=('mask', 'col_masked'), dead_weighted=('sparse', 'dead_weighted'),
    radius_open=('on_radius', dict(radius_closed=False)), no_sw=('mask', 'no_sw'),
    ray_no_z=('mask', m_ray_no_z), ray_copied=('mask', m_ray_copied),
    zero_depth_grad=('mask', 'zero_depth_grad'), no_nb_grad=('sparse', 'no_nb_grad'),
    weight_1e3=('mask', m_weight_1e3), tail64=('mask', m_tail64), pad_leak=('mask', m_pad_leak),
    upper_median=('trk_median', 'upper_median'), unc_attached=('trk_even', 'unc_attached'),
    no_suffix=('mask', 'no_suffix'))


# faults under every gate (the GPU file's docstring says why)
NOT_SEEN = {'pad_leak': (0, 1, 3), 'no_nb_grad': (0, 1, 3), 'tail64': (0, 1, 3),
            'weight_1e3': (1, 3)}


@pytest.fixture(scope='module')
def refs():
    out = {}
    for name in {v[0] for v in MUTATIONS.values()}:
        b, ctx, params, _, _ = build_ref(name)
        out[name] = dict(F.replay_step(ctx, params), batch=b)
    return out


def _mutate(refs, name):
    case, fault = MUTATIONS[name]
    ref = refs[case]
    if isinstance(fault, str):
        return ref, _remut(ref, fault)
    if isinstance(fault, dict):
        return ref, _remut(ref, **fault)
    c = _cand_of(ref)
    fault(ref, c)
    return ref, c


def test_unmutated_replay_is_clean(refs):
    for ref in refs.values():
        rep, _ = F.compare(ref, _cand_of(ref), 1e-5)
        assert max(F.worst(rep).values()) == 0.0 and rep['exempt_rows'] < 0.05


@pytest.mark.parametrize('name', sorted(MUTATIONS))
def test_mutation_is_flagged(refs, name):
    from test_pointslam_grad_f64_gpu import AMB, GATES, STRICT_MODES
    ref, cand = _mutate(refs, name)
    for mode in STRICT_MODES:
        rep, _ = F.compare(ref, cand, AMB[mode])
        assert bool(F.failures(rep, GATES[mode])) == (mode not in NOT_SEEN.get(name, ())), \
            (name, mode, F.worst(rep))


def test_mutation_floors(refs, capsys):
    """Prints the floor of every mutation (the largest ratio of the check it shows up in)."""
    with capsys.disabled():
        for name in sorted(MUTATIONS):
            ref, cand = _mutate(refs, name)
            rep, _ = F.compare(ref, cand, 1e-5)
            w = F.worst(rep)
            kind = max(('feat', 'weight', 'ray'), key=lambda k: w[k])
            per = ''
            if name == 'weight_1e3':
                per = ' min over tensors %.2g' % min(rep[k] for k in F.WEIGHT_KEYS)
            print(f'  floor {name:16s} {kind:6s} {w[kind]:.2g}{per}')
