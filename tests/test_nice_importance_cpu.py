"""NICE-SLAM stratified and importance sampling on the host: the configuration checks, the C
struct layout of the new trailing fields, and oracle/nice_importance.py against the
reference's own ConvOnet (live, when the reference checkout is present).

The reference's importance sampling passes `device=` to a sample_pdf that does not take it and
raises TypeError; the live comparisons run it under oracle.nice_importance.
sample_pdf_without_device, which drops the keyword.  The draws follow the reference's order:
torch.rand(z_vals.shape) for the jitter on the CPU generator, then sample_pdf's torch.rand."""
import ctypes as C
import warnings

import numpy as np
import pytest
import torch

from oracle import nice_importance as NI

BOUND = np.array([[-2.0, 2.0], [-2.0, 2.0], [-2.0, 2.0]])


def _model(**kw):
    from xrdslam_b200.camera import Camera
    from xrdslam_b200.conv_onet import ConvOnetConfig
    with warnings.catch_warnings():
        warnings.simplefilter('ignore', RuntimeWarning)  # no pretrained checkpoints in the tests
        return ConvOnetConfig(mapping_frustum_feature_selection=False, **kw).setup(
            camera=Camera(320., 320., 319.5, 239.5, 640, 480), bounding_box=BOUND)


@pytest.mark.parametrize('kw', [dict(rendering_perturb=1.0), dict(rendering_n_importance=16),
                                dict(rendering_n_importance=80, rendering_perturb=0.5),
                                dict(rendering_n_importance=96, coarse=True, rendering_n_surface=0)])
def test_config_accepted(kw):
    m = _model(**kw)
    assert m.config.rendering_n_importance == kw.get('rendering_n_importance', 0)


def test_config_rejected():
    with pytest.raises(NotImplementedError, match='NaN'):
        _model(rendering_lindisp=True)
    with pytest.raises(NotImplementedError, match='occupancy'):
        _model(occupancy=False)
    with pytest.raises(ValueError, match='at most 128'):
        _model(rendering_n_importance=81)             # 32 + 16 + 81
    with pytest.raises(ValueError, match='at most 128'):
        _model(rendering_n_importance=97, coarse=True, rendering_n_surface=0)
    with pytest.raises(ValueError):
        _model(rendering_n_importance=-1)


def test_struct_layout():
    """The trailing sampling fields of XrdNiceCfg and XrdNiceCoarseCfg, as the C compiler lays
    them out (x86-64: int, float, then 8-byte aligned seed and pointers)."""
    from xrdslam_b200._cabi import XrdNiceCfg, XrdNiceCoarseCfg
    for cls, base in ((XrdNiceCfg, 104), (XrdNiceCoarseCfg, 112)):
        assert cls.n_importance.offset == base, cls
        assert cls.perturb.offset == base + 4
        assert cls.seed.offset == base + 8
        assert cls.perturb_u.offset == base + 16
        assert cls.importance_u.offset == base + 24
        assert cls.t_importance.offset == base + 32
        assert C.sizeof(cls) == base + 40
    assert XrdNiceCfg.max_depth_global.offset == 96
    assert XrdNiceCoarseCfg.t_uniform.offset == 104


def test_oracle_jitter_and_merge():
    """The oracle's jitter stays in each interval and leaves the surface samples alone; the
    merge of pass 2 holds pass 1's samples and the sample_pdf draws, sorted."""
    from oracle.nice import NiceOracle
    torch.manual_seed(0)
    ora = NiceOracle(BOUND, seed=0)
    g = torch.Generator().manual_seed(1)
    R = 40
    ro = (torch.rand(R, 3, generator=g) - 0.5) * 0.6
    rd = torch.nn.functional.normalize(torch.randn(R, 3, generator=g), dim=-1)
    td = torch.rand(R, 1, generator=g) * 1.5 + 0.3
    td[::5] = 0
    noise = torch.rand(R, 32, generator=g)
    z0 = NI.sample_z(ora, ro, rd, td)
    z1 = NI.sample_z(ora, ro, rd, td, noise)
    assert bool((z1[:, 1:] >= z1[:, :-1]).all()) and not torch.equal(z0, z1)
    u = torch.rand(R, 16, generator=g)
    out = NI.render(ora, ro, rd, td, 'color', noise, u)
    assert out['z_vals'].shape == (R, 64)
    assert bool(torch.isin(z1, out['z_vals']).all())
    assert bool(torch.isin(out['z_samples'], out['z_vals']).all())


# ------------------------------------------------------------ live reference ---
def _live_pair(coarse=False, **kw):
    from oracle import ref_harness as H
    from oracle.nice import NiceOracle
    torch.manual_seed(0)
    ref = H.ref_conv_onet(BOUND, coarse=coarse, **kw)
    ora = NiceOracle(BOUND, seed=0, coarse=coarse)
    H.copy_nice_ref_to_oracle(ref, ora)
    g = torch.Generator().manual_seed(2)
    R = 24
    ro = (torch.rand(R, 3, generator=g) - 0.5) * 0.6
    rd = torch.nn.functional.normalize(torch.randn(R, 3, generator=g), dim=-1)
    td = torch.rand(R, 1, generator=g) * 1.5 + 0.3
    td[3::7] = 0
    ts = torch.rand(R, 3, generator=g)
    return ref, ora, (ro, rd, ts, td)


def _color_tensors(ref, ora, who):
    """The colour decoder's tensors in one order for both: B, pts_linears (w, b), fc_c (w, b),
    output_linear (w, b)."""
    if who == 'ref':
        d = ref.decoder.color_decoder
        t = [d.embedder._B]
        t += [x for i in range(5) for x in (d.pts_linears[i].weight, d.pts_linears[i].bias)]
        t += [x for i in range(5) for x in (d.fc_c[i].weight, d.fc_c[i].bias)]
        return t + [d.output_linear.weight, d.output_linear.bias]
    d = ora.color
    t = [d.B]
    t += [x for i in range(5) for x in (d.pts[i].weight, d.pts[i].bias)]
    t += [x for i in range(5) for x in (d.fc_c[i].weight, d.fc_c[i].bias)]
    return t + [d.out.weight, d.out.bias]


LIVE = [(0, 1.0), (5, 0.0), (16, 0.0), (5, 1.0), (16, 1.0)]


@pytest.mark.needs_reference
def test_reference_importance_raises_without_shim():
    ref, _, (ro, rd, ts, td) = _live_pair(rendering_n_importance=8)
    with pytest.raises(TypeError, match='device'):
        with torch.no_grad():
            ref.render_batch_ray(ro, rd, 'color', gt_depth=td)


@pytest.mark.needs_reference
@pytest.mark.parametrize('N,perturb', LIVE)
@pytest.mark.parametrize('stage', ['color', 'middle', 'fine', 'coarse'])
def test_oracle_matches_reference_live(N, perturb, stage):
    """Outputs, loss terms and gradients (grids, colour decoder, rays) of the oracle and of the
    reference's ConvOnet with the same draws: bit-identical."""
    from oracle import ref_harness as H
    coarse = stage == 'coarse'
    ref, ora, (ro, rd, ts, td) = _live_pair(coarse=coarse, rendering_n_importance=N,
                                            rendering_perturb=perturb)
    R = ro.shape[0]
    seed = 40 + N
    torch.manual_seed(seed)  # the reference's draws, in its order
    noise = torch.rand(R, 32) if perturb > 0 else None
    u = (torch.rand(R, N) if perturb > 0 else NI.det_u(N).expand(R, N)) if N > 0 else None
    for is_mapping in ((True,) if coarse else (True, False)):
        grads = []
        for who in ('ref', 'ora'):
            r_o = ro.clone().requires_grad_(True)
            r_d = rd.clone().requires_grad_(True)
            if who == 'ref':
                for p in ref.parameters():
                    p.grad = None
                grid = {k: v.detach().clone().requires_grad_(True) for k, v in ref.grid_c.items()}
                for k, v in grid.items():
                    ref.grid_c[k] = v
                torch.manual_seed(seed)
                with H.cuda_calls_are_noops(), NI.sample_pdf_without_device():
                    out = ref.render_batch_ray(r_o, r_d, stage, gt_depth=td)
                    ld = ref.get_loss_dict(out, dict(target_s=ts, target_d=td), is_mapping,
                                           stage) if hasattr(ref, 'get_loss_dict') else None
                gd = {k: v for k, v in grid.items()}
            else:
                for p in ora.parameters():
                    p.grad = None
                out = NI.render(ora, r_o, r_d, td, stage, noise, u)
                ld = ora.loss_dict(out, ts, td, is_mapping, stage)
                gd = {k: ora.grids[k] for k in ora.grids}
            tot = sum(ld.values())
            tot.backward()
            keys = ('rgb', 'depth', 'uncertainty') if stage == 'color' else ('depth', 'uncertainty')
            grads.append(dict(out={k: out[k].detach() for k in keys},
                              ld={k: float(v.detach()) for k, v in ld.items()},
                              grid={k: v.grad for k, v in gd.items() if v.grad is not None},
                              ro=r_o.grad, rd=r_d.grad,
                              col=[t.grad for t in _color_tensors(ref, ora, who)]
                              if stage == 'color' else []))
        a, b = grads
        for k in a['out']:
            assert torch.equal(a['out'][k], b['out'][k]), (k, is_mapping)
        assert a['ld'] == b['ld'], is_mapping
        assert set(a['grid']) == set(b['grid'])
        for k in a['grid']:
            assert torch.equal(a['grid'][k], b['grid'][k]), k
        assert torch.equal(a['ro'], b['ro']) and torch.equal(a['rd'], b['rd'])
        assert len(a['col']) == len(b['col']) == (23 if stage == 'color' else 0)
        for i, (ga, gb) in enumerate(zip(a['col'], b['col'])):
            assert (ga is None and gb is None) or torch.equal(ga, gb), (i, is_mapping)


# ------------------------------------------------------------------- mutations ---
# What a wrong sampler would produce, against the restatement: each must fail the gates the GPU
# tests apply to the device sampler (NI.sampler_failures) or the bit-exact jitter check.
def _pass1(R=200):
    from oracle.nice import NiceOracle
    with torch.random.fork_rng():
        torch.manual_seed(0)
        ora = NiceOracle(BOUND, seed=0)
    g = torch.Generator().manual_seed(5)
    with torch.no_grad():
        for k in ora.grids:
            ora.grids[k].mul_(30.0)
    ro = (torch.rand(R, 3, generator=g) - 0.5) * 0.6
    rd = torch.nn.functional.normalize(torch.randn(R, 3, generator=g), dim=-1)
    td = torch.rand(R, 1, generator=g) * 1.5 + 0.3
    td[3::7] = 0
    z1 = NI.sample_z(ora, ro, rd, td)
    with torch.no_grad():
        w = NI.render_z(ora, ro, rd, z1, 'color')['weights']
    return ora, (ro, rd, td), z1, w


def _mutant_sample_pdf(bins, weights, u, right=True, f32_bins=False):
    """oracle.coslam_importance.sample_pdf with one of its steps changed."""
    weights = weights + 1e-5
    pdf = weights / torch.sum(weights, -1, keepdim=True)
    cdf = torch.cat([torch.zeros_like(pdf[..., :1]), torch.cumsum(pdf, -1)], -1)
    if f32_bins:
        bins = bins.float()
    inds = torch.searchsorted(cdf, u.contiguous(), right=right)
    below = (inds - 1).clamp(min=0)
    above = inds.clamp(max=cdf.shape[-1] - 1)
    c0, c1 = cdf.gather(1, below), cdf.gather(1, above)
    b0, b1 = bins.gather(1, below), bins.gather(1, above)
    den = c1 - c0
    den = torch.where(den < 1e-5, torch.ones_like(den), den)
    return (b0 + (u - c0) / den * (b1 - b0)).double()


def test_mutations_fail_sampler_gates():
    _, _, z1, w = _pass1()
    R, N = z1.shape[0], 16
    mid = .5 * (z1[..., 1:] + z1[..., :-1])
    u = torch.rand(R, N, generator=torch.Generator().manual_seed(6))
    zs_o, inds, cdf = NI.sample_pdf(mid, w[..., 1:-1], u)
    ok = NI.sampler_report(zs_o, zs_o, inds, cdf, mid, u)
    assert not NI.sampler_failures(ok)
    # weights[:-2] instead of weights[1:-1]: the pdf moves by one bin
    rep = NI.sampler_report(NI.sample_pdf(mid, w[..., :-2], u)[0], zs_o, inds, cdf, mid, u)
    assert NI.sampler_failures(rep), rep
    # float32 bins: no sample stays bit-exact
    rep = NI.sampler_report(_mutant_sample_pdf(mid, w[..., 1:-1], u, f32_bins=True), zs_o, inds,
                            cdf, mid, u)
    assert NI.sampler_failures(rep), rep
    # searchsorted(right=False) differs where u equals a cdf value whose step below is under the
    # 1e-5 clamp: the sample falls a whole bin lower.  Such u are placed on the rays here.
    u2 = u.clone()
    step = cdf[:, 1:] - cdf[:, :-1]
    rows = (step[:, :-1] < 1e-5).any(-1).nonzero().squeeze(1)
    assert rows.numel() > 10
    for r in rows.tolist():
        m = int((step[r, :-1] < 1e-5).nonzero()[0]) + 1  # cdf[m] - cdf[m - 1] < 1e-5
        u2[r, 0] = cdf[r, m]
    zs2, inds2, cdf2 = NI.sample_pdf(mid, w[..., 1:-1], u2)
    rep = NI.sampler_report(_mutant_sample_pdf(mid, w[..., 1:-1], u2, right=False), zs2, inds2,
                            cdf2, mid, u2)
    assert NI.sampler_failures(rep), rep    # more samples off by a bin than the gate allows


def test_mutation_jitter_on_surface_samples_fails():
    """Jittering all 48 samples (the surface band too) changes the samples the GPU test
    requires bit for bit."""
    ora, (ro, rd, td), _, _ = _pass1(64)
    R = ro.shape[0]
    noise = torch.rand(R, 48, generator=torch.Generator().manual_seed(7))
    z_ok = NI.sample_z(ora, ro, rd, td, noise[:, :32])
    z_all = NI.jitter(NI.sample_z(ora, ro, rd, td), noise)
    z_all, _ = torch.sort(z_all, -1)
    assert not torch.equal(z_ok, z_all)


# ----------------------------------------------------------------- the fixture ---
@pytest.mark.parametrize('name', ['perturb', 'det16', 'rand16', 'fine_det5', 'coarse_rand8'])
def test_oracle_matches_reference_fixture(name):
    """The restatement against tests/golden/nice_importance_step.npz, which the reference's own
    ConvOnet wrote (tests/golden/make_golden_nice_importance.py): outputs, loss terms and the
    gradients of the grids, the colour decoder and the rays, bit for bit."""
    import os
    import sys
    here = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
    sys.path.insert(0, here)
    try:
        import make_golden_nice_importance as G
    finally:
        sys.path.remove(here)
    g = np.load(os.path.join(here, 'nice_importance_step.npz'))
    stage, is_mapping, N, perturb = G.CASES[name]
    ora = G.oracle(stage == 'coarse')
    t = lambda k: torch.from_numpy(g[k])
    ro = t('rays_o').requires_grad_(True)
    rd = t('rays_d').requires_grad_(True)
    ts, td = t('target_s'), t('target_d')
    p = name + '.'
    noise = t(p + 'noise') if p + 'noise' in g else None
    u = t(p + 'u') if p + 'u' in g else None
    out = NI.render(ora, ro, rd, td, stage, noise, u)
    ld = ora.loss_dict(out, ts, td, is_mapping, stage)
    sum(ld.values()).backward()
    for k in ('rgb', 'depth', 'uncertainty'):
        assert np.array_equal(out[k].detach().numpy(), g[p + k]), k
    assert {k for k in g if k.startswith(p + 'loss.')} == {p + 'loss.' + k for k in ld}
    for k, v in ld.items():
        assert float(v.detach()) == float(g[p + 'loss.' + k]), k
    grids = {k[len(p) + 2:] for k in g if k.startswith(p + 'd_grid')}
    assert grids == {k for k in ora.grids if ora.grids[k].grad is not None}
    for k in grids:
        assert np.array_equal(ora.grids[k].grad.numpy(), g[p + 'd_' + k]), k
    if stage == 'color':
        c = ora.color
        col = [c.B] + [x for i in range(5) for x in (c.pts[i].weight, c.pts[i].bias)] + \
            [x for i in range(5) for x in (c.fc_c[i].weight, c.fc_c[i].bias)] + \
            [c.out.weight, c.out.bias]
        for i, x in enumerate(col):
            assert np.array_equal(x.grad.numpy(), g[p + f'd_color{i}']), i
    assert np.array_equal(ro.grad.numpy(), g[p + 'd_rays_o'])
    assert np.array_equal(rd.grad.numpy(), g[p + 'd_rays_d'])


def test_seed_advances_and_differs_per_rank():
    """Without explicit uniforms the kernels draw from XrdNiceCfg.seed: it advances every
    launch, and ranks of data-parallel mapping (same step count) draw from different seeds."""
    from types import SimpleNamespace

    from xrdslam_b200._cabi import XrdNiceCfg
    m = _model(rendering_n_importance=16, rendering_perturb=1.0)
    seeds = []
    for rank in (0, 0, 1):
        m.dp = SimpleNamespace(rank=rank) if rank else None
        c = XrdNiceCfg()
        assert m._sampling(c, 10, 48, None, None, 'cpu', []) == 64
        assert c.n_importance == 16 and c.perturb == 1.0 and not c.perturb_u
        seeds.append(c.seed)
    assert seeds[0] != seeds[1]
    m2 = _model(rendering_n_importance=16, rendering_perturb=1.0)
    m2._step_count = 1
    m2.dp = SimpleNamespace(rank=1)
    c = XrdNiceCfg()
    m2._sampling(c, 10, 48, None, None, 'cpu', [])
    assert c.seed not in seeds[:2]          # rank 1 at step 2 differs from rank 0 at step 2
