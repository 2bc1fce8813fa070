"""The float64 Vox-Fusion replay (oracle/voxfusion_f64.py) and its checker, on the CPU.

- The replay agrees with the fp32 oracle (oracle/voxfusion.py VoxOracle.render) at fp32 level:
  outputs, loss terms and every gradient, and the fp32 oracle passes the GPU gates of every mode.
- gradcheck of the replay on a 3-ray batch pins the dp/d(o, d) carrier, the corner weights and
  the loss normalisers.
- Mutations of the fp32 oracle's gradient that a kernel bug would produce are flagged at the
  gates test_voxfusion_grad_f64_gpu.py applies to GEMM modes 0, 1 and 3.  The smallest ratio
  each produces (its floor, on the scene case below) is in the GPU file's table.
"""
import pytest
import torch

from oracle import voxfusion_f64 as F
from test_voxfusion_cpu import vox_oracle_case
from test_voxfusion_grad_f64_gpu import AMB, GATES

# what fp32 arithmetic leaves against float64 (worst seen on the CPU: entry 4e-9, weight 2.4e-7,
# ray 1.1e-10, loss 1.1e-7, forward 2.6e-7)
FP32_GATES = dict(entry=1e-7, weight=1e-6, ray=1e-8, loss=1e-6, fwd=1e-6)
STRICT_MODES = (0, 1, 3)


def _dec_params(ora):
    d = ora.decoder
    return [d.pts_linears[0].weight, d.pts_linears[0].bias, d.pts_linears[1].weight,
            d.pts_linears[1].bias, d.sdf_out.weight, d.sdf_out.bias, d.color_out[0].weight,
            d.color_out[0].bias, d.color_out[2].weight, d.color_out[2].bias]


def _scene_case(R=300):
    """A few hundred rays of the GPU tests' scene (map built by the package's host octree),
    embeddings randn * 0.3, some rays of more than 64 samples.  The sdf bias is lifted to the
    median sample sdf, so that many rays change sign inside their samples, not only at the
    padded tail (sdf 1)."""
    from oracle.voxfusion import VoxOracle
    from test_voxfusion_gpu import scene
    model, ro, rd, ts, td = scene('cpu', R=R, seed=4)
    ora = VoxOracle()
    with torch.no_grad():
        g = torch.Generator().manual_seed(9)
        ora.embeddings.copy_(torch.randn(model.embeddings.shape, generator=g) * 0.3)
        ora.decoder.load_state_dict(model.decoder.state_dict())
    ora.set_map(*model.export_octree())
    gen = torch.Generator().manual_seed(5)
    marched = ora.march(ro, rd, lambda s: torch.rand(s, generator=gen).clamp(0.001, 0.999))
    with torch.no_grad():
        out, _ = ora.render(ro, rd, None, None, marched)
        valid = marched[2]['sampled_point_voxel_idx'] >= 0
        ora.decoder.sdf_out.bias[0] -= float(out['sdf'][valid].median())
    return ora, marched, (ro, rd, ts, td)


def _step(case):
    """fp32 oracle gradients (the candidate) and the float64 replay of the same step."""
    ora, marched, (ro, rd, ts, td) = case
    ro_o, rd_o = ro.clone().requires_grad_(True), rd.clone().requires_grad_(True)
    out, ld = ora.render(ro_o, rd_o, ts, td, marched)
    sum(ld.values()).backward()
    dec = _dec_params(ora)
    cand = dict(d_emb=ora.embeddings.grad, d_dec=[t.grad for t in dec], d_rays_o=ro_o.grad,
                d_rays_d=rd_o.grad, losses=torch.stack([v.detach() for v in ld.values()]),
                rgb=out['rgb'].detach(), depth=out['depth'].detach())
    cand = {k: ([t.double() for t in v] if isinstance(v, list) else v.double())
            for k, v in cand.items()}
    ctx = F.prepare(ro, rd, ts, td, F.from_oracle(marched, ro.shape[0]), ora.centres,
                    ora.vertex_idx, ora.voxel_size, ora.trunc, ora.max_depth, 10.0, ora.w)
    ref = F.replay_step(ctx, ora.embeddings, dec)
    return ora, ref, cand, out['sdf'].detach()


@pytest.fixture(scope='module')
def small():
    return _step(vox_oracle_case())


@pytest.fixture(scope='module')
def step():
    return _step(_scene_case())


def test_scene_case_shape(step):
    _, ref, _, sdf = step
    ctx = ref['ctx']
    change = ((sdf[:, 1:] * sdf[:, :-1]) < 0).any(1)
    inner = change & (ref['first'] + 1 < ctx['count'])      # a sign change inside the samples
    assert int(inner.sum()) > ctx['Rh'] // 4 and bool((~change).any())
    assert bool((ctx['count'] > 64).any()) and bool((ctx['count'] < ctx['S']).any())
    assert not bool(ctx['ray_mask'].all())


@pytest.mark.parametrize('case', ['small', 'step'])
def test_replay_matches_fp32_oracle(case, request):
    _, ref, cand, sdf = request.getfixturevalue(case)
    rep = F.compare(ref, cand, AMB[0], sdf)
    assert rep['n_flip_rays'] == 0
    assert not F.failures(rep, FP32_GATES), F.failures(rep, FP32_GATES)


@pytest.mark.parametrize('mode', [0, 1, 2, 3])
@pytest.mark.parametrize('case', ['small', 'step'])
def test_fp32_oracle_passes_gpu_gates(case, mode, request):
    _, ref, cand, sdf = request.getfixturevalue(case)
    assert not F.failures(F.compare(ref, cand, AMB[mode], sdf), GATES[mode])


def test_gradcheck_replay():
    """With the discrete inputs frozen the replay is smooth: its analytic float64 gradients with
    respect to the rays, the sdf-head weights and the embedding rows of the batch match finite
    differences."""
    ora, marched, (ro, rd, ts, td) = vox_oracle_case()
    hits = marched[1]
    keep = torch.nonzero(hits).reshape(-1)[[0, 7, 20]]
    sub = torch.zeros_like(hits)
    sub[keep] = True
    inter, _, smp = marched
    sel = hits.cumsum(0)[keep] - 1
    smp3 = {k: (v[sel] if torch.is_tensor(v) and v.dim() and v.shape[0] == hits.sum() else v)
            for k, v in smp.items()}
    S = int((smp3['sampled_point_voxel_idx'] >= 0).sum(1).max())
    smp3 = {k: (v[:, :S] if torch.is_tensor(v) and v.dim() == 2 else v) for k, v in smp3.items()}
    R = 3
    ro3, rd3, ts3, td3 = ro[keep], rd[keep], ts[keep], td[keep].clone()
    td3[1] = 0.005                 # one ray outside the valid-depth range: normalisers change
    m3 = (None, torch.ones(R, dtype=torch.bool), smp3)
    ctx = F.prepare(ro3, rd3, ts3, td3, F.from_oracle(m3, R), ora.centres, ora.vertex_idx)
    dec0 = [t.detach().double() for t in _dec_params(ora)]
    emb0 = ora.embeddings.detach().double()
    rows = torch.unique(ctx['vid'].reshape(-1))[:6]
    f0 = F.forward(ctx, ro3.double(), rd3.double(), emb0, dec0, leaf=False)
    first = f0['first']

    def fn(ro_, rd_, e_rows, ws, bs):
        emb = emb0.index_put((rows,), e_rows)
        dec = dec0[:4] + [ws, bs] + dec0[6:]
        return F.forward(ctx, ro_, rd_, emb, dec, first=first, leaf=False)['total']

    args = (ro3.double().requires_grad_(True), rd3.double().requires_grad_(True),
            emb0[rows].clone().requires_grad_(True), dec0[4].clone().requires_grad_(True),
            dec0[5].clone().requires_grad_(True))
    assert torch.autograd.gradcheck(fn, args, eps=1e-6, atol=1e-7, rtol=1e-5)


# ---- mutations: what a wrong kernel would produce, applied to the fp32 oracle's gradient ----
def _flagged_ratio(ref, mut, sdf, modes=STRICT_MODES):
    """The report of the mutated candidate at the mode-0 threshold, after asserting that every
    strict mode's gates flag it."""
    for m in modes:
        assert F.failures(F.compare(ref, mut, AMB[m], sdf), GATES[m]), m
    return F.compare(ref, mut, AMB[0], sdf)


def _busiest_voxel(ref):
    """Points of the voxel with the most points among those whose corner rows no ReLU-ambiguous
    point touches (such rows leave the per-entry check)."""
    ctx = ref['ctx']
    vox, vid = ctx['vox'], ctx['vid']
    _, amb = F.flip_bounds(ref, AMB[1])
    touched = torch.zeros(ref['emb'].shape[0], dtype=torch.bool)
    touched[vid[amb].reshape(-1)] = True
    clean = ~touched[vid].any(1)
    v, n = torch.unique(vox[clean], return_counts=True)
    pts = torch.nonzero(vox == v[n.argmax()]).reshape(-1)
    assert bool(clean[pts].all()) and len(pts) > 20
    return pts


def _emb_add(g, ref, pts, wdelta):
    """g[vid_i] += wdelta[p, i] * dx[p] for p in pts."""
    out = g.clone()
    vid = ref['ctx']['vid'][pts]
    out.index_add_(0, vid.reshape(-1), (wdelta[..., None] * ref['dx'][pts][:, None, :]).reshape(-1, 16))
    return out


def test_mutation_corner_takes_x_neighbour(step):
    """Corner 0 of one voxel scattered to the vertex of corner 0 ^ 4 (its x-neighbour)."""
    _, ref, cand, sdf = step
    pts = _busiest_voxel(ref)
    w0 = ref['wc'][pts, 0]
    g = _emb_add(cand['d_emb'], ref, pts, torch.nn.functional.one_hot(
        torch.zeros(len(pts), dtype=torch.long), 8).double() * -w0[:, None])
    vid4 = ref['ctx']['vid'][pts, 4]
    g.index_add_(0, vid4, w0[:, None] * ref['dx'][pts])
    _flagged_ratio(ref, dict(cand, d_emb=g), sdf)


def test_mutation_axis_weight_from_other_axis(step):
    """The trilinear weights of one voxel built with p_y in place of p_x."""
    _, ref, cand, sdf = step
    pts = _busiest_voxel(ref)
    p = ref['p'][pts].clone()
    p[:, 0] = p[:, 1]
    g = _emb_add(cand['d_emb'], ref, pts, F.corner_weights(p) - ref['wc'][pts])
    _flagged_ratio(ref, dict(cand, d_emb=g), sdf)


# (weight key, its activation input, its pre-activation gradient) per decoder layer
LAYERS = {'w0': ('x', 'dpre1'), 'w1': ('h1', 'dpre2'), 'ws': ('h2', 'dso'),
          'wc0': ('inc', 'dprec'), 'wc1': ('c1', 'draw')}


@pytest.mark.parametrize('key', list(LAYERS))
def test_mutation_drop_last_64_points(step, key):
    """The last 64 points missing from one weight gradient and its bias (a lost k_dw_tc
    staging tail)."""
    _, ref, cand, sdf = step
    a, b = LAYERS[key]
    A, B = ref[a][-64:], ref[b][-64:]
    if key == 'wc1':
        B = B[:, :3]
    i = F.DEC_KEYS.index(key)
    dec = list(cand['d_dec'])
    dec[i] = dec[i] - B.T @ A
    dec[i + 1] = dec[i + 1] - B.sum(0)
    _flagged_ratio(ref, dict(cand, d_dec=dec), sdf)


def test_mutation_wc0_x_columns_zero(step):
    """wc0 columns 128..143 (the x half of the colour input, its own k_dw job) zero."""
    _, ref, cand, sdf = step
    dec = list(cand['d_dec'])
    dec[6] = dec[6].clone()
    dec[6][:, 128:] = 0
    _flagged_ratio(ref, dict(cand, d_dec=dec), sdf)


@pytest.mark.parametrize('key', ['w0', 'w1', 'ws', 'wc0', 'wc1'])
def test_mutation_scale_one_element(step, key):
    """One element of one weight gradient scaled by 1 + 1e-3: the element whose value is largest
    against its bound A (elements whose terms cancel to far below A cannot show it)."""
    _, ref, cand, sdf = step
    i = F.DEC_KEYS.index(key)
    dec = list(cand['d_dec'])
    g = dec[i].clone().reshape(-1)
    A = F.abs_bounds(ref)['d_' + key].reshape(-1)
    e = int((ref['grads']['d_' + key].abs().reshape(-1) / A.clamp_min(1e-300)).argmax())
    g[e] *= 1 + 1e-3
    dec[i] = g.reshape(dec[i].shape)
    # w0, ws and wc1 reach 6.4e-6, 2.5e-6 and 1e-6: flagged by the fp32 gate of mode 0 only
    _flagged_ratio(ref, dict(cand, d_dec=dec), sdf,
                   modes=STRICT_MODES if key in ('w1', 'wc0') else (0,))


@pytest.mark.parametrize('which', ['smallest', 'largest'])
@pytest.mark.parametrize('key', ['d_rays_o', 'd_rays_d'])
def test_mutation_copy_neighbour_ray(step, which, key):
    _, ref, cand, sdf = step
    mag = ref['grads'][key].norm(dim=1)
    hit = torch.nonzero(ref['ctx']['ray_mask']).reshape(-1)
    r = int(hit[mag[hit].argmin()] if which == 'smallest' else hit[mag[hit].argmax()])
    src = r - 1 if r > 0 else r + 1
    g = cand[key].clone()
    g[r] = g[src]
    _flagged_ratio(ref, dict(cand, **{key: g}), sdf)


def test_mutation_rays_d_without_z(step):
    """d_rays_d of one ray summed without the depth factor (= its d_rays_o)."""
    _, ref, cand, sdf = step
    r = int(ref['grads']['d_rays_d'].norm(dim=1).argmax())
    g = cand['d_rays_d'].clone()
    g[r] = cand['d_rays_o'][r]
    _flagged_ratio(ref, dict(cand, d_rays_d=g), sdf)


def _replay_delta(ora, ref, **kw):
    """Gradient of the replay with a changed rule minus the replay's own."""
    alt = F.replay_step(ref['ctx'], ora.embeddings, _dec_params(ora), **kw)['grads']
    return {k: alt[k] - ref['grads'][k] for k in alt}


def _apply(cand, delta):
    out = dict(cand)
    out['d_emb'] = cand['d_emb'] + delta['d_emb']
    out['d_dec'] = [t + delta[k].reshape(t.shape) for t, k in zip(cand['d_dec'], F.WEIGHT_KEYS)]
    for k in F.RAY_KEYS:
        out[k] = cand[k] + delta[k]
    return out


def test_mutation_zlim_shifted_one_sample(step):
    """One ray's truncation window z < z[first] + tr taken one sample later."""
    ora, ref, cand, sdf = step
    ctx = ref['ctx']
    tm = F.trunc_mask(ctx, ref['first'])
    for r in torch.nonzero(ref['first'] + 1 < ctx['count']).reshape(-1).tolist():
        first = ref['first'].clone()
        first[r] += 1
        if not torch.equal(F.trunc_mask(ctx, first), tm):
            break
    assert not torch.equal(F.trunc_mask(ctx, first), tm)
    _flagged_ratio(ref, _apply(cand, _replay_delta(ora, ref, first=first)), sdf)


def test_mutation_q3_per_ray_normaliser(step):
    """The sdf / fs means over Rh * count[r] instead of the batch-wide Rh * S (SURVEY Q3)."""
    ora, ref, cand, sdf = step
    assert bool((ref['ctx']['count'] < ref['ctx']['S']).any())
    _flagged_ratio(ref, _apply(cand, _replay_delta(ora, ref, per_ray_norm=True)), sdf)
