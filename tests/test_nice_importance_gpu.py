"""NICE-SLAM stratified and importance sampling on the device (rendering_perturb > 0,
rendering_n_importance > 0) against oracle/nice_importance.py, itself pinned to the
reference's ConvOnet (tests/test_nice_importance_cpu.py).

  sampler  xrd_nice_sample_pdf on the oracle's pass-1 weights and samples: the merged samples
           match the oracle's sample_pdf and sort to 1e-3 (see test_sampler_bit_exact), for
           the det draw and a given u;
           the Philox draw is deterministic per seed, fresh across seeds and uniform
  jitter   with the uniforms given, the jittered samples of the step and of the coarse step are
           bit-exact to the oracle's
  step     the kernel's merged samples run through the oracle's pass 2, judged per grid entry,
           per colour-decoder element and per ray with ``report`` and the gates of
           test_nice_noncubic_gpu.py, on its non-cubic bound; N = 80 reaches 128 samples
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import nice_importance as NI
from test_nice_gpu import nice_pair
from test_nice_noncubic_gpu import BOUND_NC, GATES, _rays, failures, report

pytestmark = pytest.mark.gpu

# test_nice_noncubic_gpu.py's gates up to 64 samples per ray.  Above, the ray gate is raised: the
# worst ray ratio observed on an H100 80GB HBM3 was 1.6e-3 (colour, mapping, N = 80, det draw),
# where the det quantiles put many samples within a few ulps of each other.
GATES_128 = dict(GATES, ray=4e-3)


def gates(S):
    return GATES if S <= 64 else GATES_128


# the step's merged samples against the restatement's own (NI.merged_offsets, in pass-1 bin
# widths): pass 1's weights differ from torch's by float ulps, so a sample moves by ulps of the
# cdf over its step; at most this fraction of the merged values may be off by 1e-3 bin widths
MERGE_BAD = 5e-3


def configure(model, n_importance, perturb):
    """Set the sampling options of a built model (nice_pair builds the default config)."""
    cfg = model.config
    cfg.rendering_n_importance, cfg.rendering_perturb = n_importance, perturb
    n = max(n_importance, 1)
    model._t_importance = torch.linspace(0. + 0.5 / n, 1. - 0.5 / n, steps=n).to(
        model._t_uniform.device)
    return model


def draws(R, ns, N, perturb, seed):
    """(noise [R, ns] or None, u [R, N] or None) in the reference's order: the jitter's
    torch.rand first, then sample_pdf's (or its det linspace when perturb == 0)."""
    g = torch.Generator().manual_seed(seed)
    noise = torch.rand(R, ns, generator=g) if perturb > 0 else None
    u = None
    if N > 0:
        u = torch.rand(R, N, generator=g) if perturb > 0 else NI.det_u(N).expand(R, N)
    return noise, u


def kernel_sample_pdf(w, z, N, u=None, det=False, seed=0, z_samples=None):
    from xrdslam_b200 import _cabi
    dev = w.device
    R, S0 = w.shape
    out = torch.empty(R, S0 + N, dtype=torch.float64, device=dev)
    n = max(N, 1)
    lin = torch.linspace(0. + 0.5 / n, 1. - 0.5 / n, steps=n).to(dev)
    from xrdslam_b200._cabi import ptr
    _cabi.launch_on(dev, 'xrd_nice_sample_pdf', R, S0, N, ptr(w.contiguous()),
                    ptr(z.contiguous()), ptr(u.contiguous() if u is not None else None),
                    ptr(lin), int(det), C.c_uint64(seed), ptr(out), ptr(z_samples))
    torch.cuda.synchronize()
    return out


def _pass1(R=300, seed=3, perturb=0.0):
    ora, _ = nice_pair('cpu', bound=BOUND_NC)
    ro, rd, ts, td = _rays('odd')
    noise, _ = draws(ro.shape[0], 32, 0, perturb, seed)
    z1 = NI.sample_z(ora, ro, rd, td, noise)
    with torch.no_grad():
        p1 = NI.render_z(ora, ro, rd, z1, 'color')
    return z1, p1['weights']


@pytest.mark.parametrize('N', [5, 16, 80])
@pytest.mark.parametrize('det', [True, False])
def test_sampler_matches_oracle(cuda_dev, N, det):
    """xrd_nice_sample_pdf on the restatement's pass-1 weights and samples.  The pdf's
    normaliser is the float64 sum rounded once, one float32 ulp off torch's vectorised float32
    sum on some rays; the samples of the other rays are bit-exact, the rest agree to 1e-3 of
    their bin unless that ulp is amplified (NI.sampler_report).  The merge is the sorted union."""
    z1, w = _pass1()
    R = z1.shape[0]
    u = NI.det_u(N).expand(R, N) if det else torch.rand(R, N, generator=torch.Generator().manual_seed(N))
    z_mid = .5 * (z1[..., 1:] + z1[..., :-1])
    smp, inds, cdf = NI.sample_pdf(z_mid, w[..., 1:-1], u)
    zs = torch.empty(R, N, dtype=torch.float64, device=cuda_dev)
    got = kernel_sample_pdf(w.to(cuda_dev), z1.to(cuda_dev), N,
                            None if det else u.to(cuda_dev), det=det, z_samples=zs).cpu()
    zs = zs.cpu()
    rep = NI.sampler_report(zs, smp, inds, cdf, z_mid, u)
    print('sampler', N, det, rep)
    assert not NI.sampler_failures(rep), rep
    assert torch.equal(got, torch.sort(torch.cat([z1, zs], -1), -1)[0])


def test_sampler_philox(cuda_dev):
    """Philox draws: the same seed gives the same samples, another seed others; the draws are
    uniform (one KS test)."""
    from scipy import stats
    R, S0, N = 512, 48, 64
    w = torch.zeros(R, S0, device=cuda_dev)           # pdf of 1e-5 everywhere: flat
    z = torch.linspace(0, 1, S0, dtype=torch.float64).expand(R, S0).contiguous()
    zd = z.to(cuda_dev)
    a = kernel_sample_pdf(w, zd, N, seed=11)
    b = kernel_sample_pdf(w, zd, N, seed=11)
    c = kernel_sample_pdf(w, zd, N, seed=12)
    assert torch.equal(a, b)
    assert not torch.equal(a, c)
    # the importance samples are the values not among z; on a flat pdf over evenly spaced
    # bins [mid_0, mid_last] they are lo + u (hi - lo)
    zs = z[0].numpy()
    allx = np.concatenate([np.setdiff1d(a[r].cpu().numpy(), zs) for r in range(R)])
    lo, hi = 0.5 * (zs[0] + zs[1]), 0.5 * (zs[-2] + zs[-1])
    assert allx.size > R * N * 0.99
    p = stats.kstest((allx - lo) / (hi - lo), 'uniform').pvalue
    assert p > 1e-3, p


@pytest.mark.parametrize('coarse', [False, True])
def test_jitter_bit_exact(cuda_dev, coarse):
    ora, model = nice_pair(cuda_dev, bound=BOUND_NC, coarse=coarse)
    configure(model, 0, 1.0)
    ro, rd, ts, td = _rays('odd')
    R = ro.shape[0]
    noise, _ = draws(R, 32, 0, 1.0, 7)
    S = 32 if coarse else 48
    z = torch.empty(R, S, dtype=torch.float64, device=cuda_dev)
    model._z_capture = z
    stage = 'coarse' if coarse else 'middle'
    with torch.no_grad():
        model(dict(rays_o=ro.to(cuda_dev), rays_d=rd.to(cuda_dev), target_s=None,
                   target_d=td.to(cuda_dev), stage=stage, noise=noise.to(cuda_dev)))
    torch.cuda.synchronize()
    z_o = NI.sample_z(ora, ro, rd, None if coarse else td, noise)
    assert torch.equal(z.cpu(), z_o)
    assert not torch.equal(z_o, NI.sample_z(ora, ro, rd, None if coarse else td))


def oracle_step(ora, stage, is_mapping, ro, rd, ts, td, noise, u, z):
    for p in ora.parameters():
        p.grad = None
    ro = ro.detach().clone().requires_grad_(True)
    rd = rd.detach().clone().requires_grad_(True)
    out, ld, tot = NI.step(ora, ro, rd, ts, td, is_mapping, stage, noise, u, z_fine=z)
    tot.backward()
    c = ora.color
    col = [c.B]
    for i in range(5):
        col += [c.pts[i].weight, c.pts[i].bias]
    for i in range(5):
        col += [c.fc_c[i].weight, c.fc_c[i].bias]
    col += [c.out.weight, c.out.bias]
    return dict(grids={k: ora.grids[k].grad.squeeze(0).permute(1, 2, 3, 0)
                       for k in ora.grids if ora.grids[k].grad is not None},
                color=[t.grad for t in col] if stage == 'color' else None,
                d_rays_o=ro.grad, d_rays_d=rd.grad,
                fwd={k: out[k].detach() for k in ('rgb', 'depth', 'uncertainty')},
                losses={k: float(v.detach()) for k, v in ld.items()}, out=out)


def model_step(model, stage, is_mapping, ro, rd, ts, td, noise, u, S, dev):
    z = torch.empty(ro.shape[0], S, dtype=torch.float64, device=dev)
    model._z_capture = z
    rk = ro.detach().to(dev).requires_grad_(True)
    dk = rd.detach().to(dev).requires_grad_(True)
    inp = dict(rays_o=rk, rays_d=dk, target_s=ts.to(dev), target_d=td.to(dev), stage=stage,
               is_mapping=is_mapping)
    if noise is not None:
        inp['noise'] = noise.to(dev)
    if u is not None:
        inp['importance_u'] = u.to(dev)
    out = model(inp)
    ld = model.get_loss_dict(out, inp, is_mapping, stage)
    sum(ld.values()).backward()
    torch.cuda.synchronize()
    cpu = lambda t: t.detach().cpu()
    return dict(grids={k: cpu(v.grad) for k, v in model.grids.items() if v.grad is not None},
                color=[cpu(t.grad) for t in model.decoder.color_decoder.tensors()]
                if stage == 'color' else None,
                d_rays_o=cpu(rk.grad), d_rays_d=cpu(dk.grad),
                fwd={k: cpu(out[k]) for k in ('rgb', 'depth', 'uncertainty')},
                losses={k: float(v.detach()) for k, v in ld.items()}, z=z.cpu())


def case(dev, stage, is_mapping, N, perturb, rays='odd'):
    coarse = stage == 'coarse'
    ora, model = nice_pair(dev, bound=BOUND_NC, coarse=coarse)
    configure(model, N, perturb)
    ro, rd, ts, td = _rays(rays)
    R = ro.shape[0]
    noise, u = draws(R, 32, N, perturb, 100 + N)
    S0 = 32 if coarse else 48
    # the det draw comes from the model's linspace table (no u given), the random one is given
    cand = model_step(model, stage, is_mapping, ro, rd, ts, td, noise,
                      u if perturb > 0 else None, S0 + N, dev)
    # the step's own samples against the restatement's two passes (no z_fine)
    z1 = NI.sample_z(ora, ro, rd, None if coarse else td, noise)
    with torch.no_grad():
        z_o = NI.render(ora, ro, rd, td, stage, noise, u)['z_vals']
    assert bool(torch.isin(z1, cand['z']).all())         # pass 1's samples pass through
    off = NI.merged_offsets(cand['z'], z_o, z1)
    bad = float((off > 1e-3).double().mean())
    print(f'merge: {bad:.3g} of the values off by > 1e-3 bins, median {float(off.median()):.3g}')
    assert bad < MERGE_BAD, bad
    ref = oracle_step(ora, stage, is_mapping, ro, rd, ts, td, noise, u, cand['z'])
    return report(ref, cand), ref, cand


CASES = [(st, m, N, pt) for st in ('middle', 'fine', 'color') for m in (True, False)
         for N in (8, 80) for pt in (0.0, 1.0)]


@pytest.mark.parametrize('stage,is_mapping,N,perturb', CASES)
def test_step_vs_oracle(cuda_dev, stage, is_mapping, N, perturb):
    rep, _, _ = case(cuda_dev, stage, is_mapping, N, perturb)
    print(stage, is_mapping, N, perturb, rep)
    bad = failures(rep, gates(48 + N))
    assert not bad, (bad, rep)


@pytest.mark.parametrize('N,perturb', [(8, 0.0), (16, 1.0), (96, 1.0)])
def test_coarse_step_vs_oracle(cuda_dev, N, perturb):
    rep, _, _ = case(cuda_dev, 'coarse', True, N, perturb)
    print('coarse', N, perturb, rep)
    bad = failures(rep, gates(32 + N))
    assert not bad, (bad, rep)


def test_forward_only_matches_oracle(cuda_dev):
    """The forward-only launch (render_img) with importance and the det draw from the model's
    table: the samples agree with the restatement's two passes, and pass 2's maps with the
    oracle's on the kernel's samples."""
    ora, model = nice_pair(cuda_dev, bound=BOUND_NC)
    configure(model, 16, 0.0)
    ro, rd, ts, td = _rays('default')
    R = ro.shape[0]
    z = torch.empty(R, 64, dtype=torch.float64, device=cuda_dev)
    model._z_capture = z
    with torch.no_grad():
        out = model(dict(rays_o=ro.to(cuda_dev), rays_d=rd.to(cuda_dev), target_s=None,
                         target_d=td.to(cuda_dev), stage='color'))
        ref = NI.render_z(ora, ro, rd, z.cpu(), 'color')
        z_o = NI.render(ora, ro, rd, td, 'color', None, NI.det_u(16).expand(R, 16))['z_vals']
    off = NI.merged_offsets(z.cpu(), z_o, NI.sample_z(ora, ro, rd, td))
    assert float((off > 1e-3).double().mean()) < MERGE_BAD
    for k in ('rgb', 'depth', 'uncertainty'):
        assert float((out[k].cpu().double() - ref[k].double()).abs().max()) < GATES['fwd'], k


def test_limits(cuda_dev):
    """129 samples are refused by the model, 128 run; rendering_lindisp keeps raising."""
    from xrdslam_b200.camera import Camera
    from xrdslam_b200.conv_onet import ConvOnetConfig
    cam = Camera(320., 320., 319.5, 239.5, 640, 480)
    with pytest.raises(ValueError, match='128'):
        ConvOnetConfig(rendering_n_importance=81).setup(camera=cam, bounding_box=BOUND_NC)
    rep, _, cand = case(cuda_dev, 'color', True, 80, 1.0)
    assert cand['z'].shape[1] == 128 and bool(torch.isfinite(cand['fwd']['depth']).all())


def test_seeded_draws_advance(cuda_dev):
    """Without explicit uniforms, every launch draws from a fresh seed: two launches on the same
    rays give different samples, each finite."""
    _, model = nice_pair(cuda_dev, bound=BOUND_NC)
    configure(model, 16, 1.0)
    ro, rd, ts, td = _rays('odd')
    zs = []
    for _ in range(2):
        z = torch.empty(ro.shape[0], 64, dtype=torch.float64, device=cuda_dev)
        model._z_capture = z
        with torch.no_grad():
            out = model(dict(rays_o=ro.to(cuda_dev), rays_d=rd.to(cuda_dev), target_s=None,
                             target_d=td.to(cuda_dev), stage='color'))
        torch.cuda.synchronize()
        assert bool(torch.isfinite(out['depth']).all())
        zs.append(z.cpu())
    assert not torch.equal(zs[0], zs[1])
    assert bool((zs[0][:, 1:] >= zs[0][:, :-1]).all())
