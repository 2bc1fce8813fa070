"""The float64 Co-SLAM replay (oracle/coslam_f64.py) and its checker, on the CPU.

- The replay agrees with the fp32 oracle at fp32 level per hash level, per entry, per weight
  element, per ray and per loss term, and the fp32 oracle passes the GPU gates of every mode.
- gradcheck of the replay on a 3-ray batch pins the dw/dx carrier and the loss normalisers.
- Mutations of the fp32 oracle's gradient that a kernel bug would produce are flagged at the
  gates test_coslam_grad_f64_gpu.py applies to precision modes 0 and 1.
"""
import numpy as np
import pytest
import torch

from helpers import BOUND, make_rays
from oracle import coslam_f64 as F
from test_coslam_grad_f64_gpu import AMB, GATES

# what fp32 arithmetic leaves against float64 (worst seen on the CPU: level 4.5e-7,
# entry 1.7e-7, weight 1e-9, ray 3e-9, loss 1e-7)
FP32_GATES = dict(level=2e-6, entry=1e-6, weight=1e-8, ray=2e-8, loss=1e-6)


def _oracle(amp, seed=1):
    from oracle.coslam import CoslamOracle
    ora = CoslamOracle(BOUND)
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        ora.embed_fn.params.copy_((torch.rand(ora.embed_fn.params.shape, generator=g) * 2 - 1)
                                  * amp)
        for lin in (ora.sdf0, ora.sdf1, ora.col0, ora.col1):
            lin.weight.copy_(torch.randn(lin.weight.shape, generator=g)
                             / np.sqrt(lin.weight.shape[1]))
    return ora


@pytest.fixture(scope='module')
def step4097():
    """The one-ray-final-unit batch at table amplitude 0.1: fp32 oracle gradients and the
    float64 replay of the same step."""
    R = 4097
    ora = _oracle(0.1)
    ro, rd, ts, td, noise = make_rays(R, seed=R)
    ro.requires_grad_(True)
    rd.requires_grad_(True)
    out, ld, tot = ora.step(ro, rd, ts, td, noise, False, True)
    tot.backward()
    cand = dict(d_table=ora.embed_fn.params.grad, d_w_sdf0=ora.sdf0.weight.grad,
                d_w_sdf1=ora.sdf1.weight.grad, d_w_col0=ora.col0.weight.grad,
                d_w_col1=ora.col1.weight.grad, d_rays_o=ro.grad, d_rays_d=rd.grad,
                losses=torch.stack([ld[k].detach() for k in
                                    ('rgb_loss', 'depth_loss', 'sdf_loss', 'fs_loss')]))
    cand = {k: v.detach().double() for k, v in cand.items()}
    ref = F.replay_step(ora, ro, rd, ts, td, out['z_vals'])
    return ora, ref, cand, out['raw'][..., 3].detach()


def _flagged(ref, cand, sdf, modes=(0, 1)):
    """Modes at whose gates the candidate is NOT flagged."""
    return [m for m in modes if not F.failures(F.compare(ref, cand, AMB[m], sdf), GATES[m])]


def test_fp32_oracle_within_fp32_of_float64(step4097):
    _, ref, cand, sdf = step4097
    rep = F.compare(ref, cand, AMB[0], sdf)
    assert rep['n_flip_rays'] == 0
    assert rep['n_amb_points'] < ref['R'] * ref['S'] // 100
    assert not F.failures(rep, FP32_GATES), F.failures(rep, FP32_GATES)


@pytest.mark.parametrize('mode', [0, 1, 2])
def test_fp32_oracle_passes_gpu_gates(step4097, mode):
    _, ref, cand, sdf = step4097
    assert not F.failures(F.compare(ref, cand, AMB[mode], sdf), GATES[mode])


def test_gradcheck_replay():
    """With the discrete inputs frozen the replay is smooth: its analytic float64 gradients
    with respect to the rays, the weights and a few table entries match finite differences."""
    R = 3
    ora = _oracle(0.3, seed=4)
    ro, rd, ts, td, noise = make_rays(R, seed=9, zero_depth_every=0)
    td[1] = 0                          # one ray without depth: the loss normalisers change
    z = ora.sample_z(R, td, noise)
    ctx = F.prepare(ora, ro, rd, ts, td, z)
    table0 = ora.embed_fn.params.detach().double()
    Ws0 = [lin.weight.detach().double() for lin in (ora.sdf0, ora.sdf1, ora.col0, ora.col1)]
    f0 = F.forward(ctx, ro.double(), rd.double(), table0.clone().requires_grad_(True),
                   [w.clone().requires_grad_(True) for w in Ws0])
    inds = f0['inds']
    # a handful of entries the batch touches, on a coarse and on a fine level
    touched = torch.unique(ctx['idx'][:, [0, 14], :].reshape(-1))
    sel = torch.cat([touched[:3] * 2, touched[-3:] * 2 + 1])
    scale = (0.5, 2.0, 1.5, 0.25)

    def fn(ro_, rd_, sub, w0, w1, wc0, wc1):
        table = table0.index_put((sel,), sub)
        return F.forward(ctx, ro_, rd_, table, [w0, w1, wc0, wc1], scale, inds=inds)['total']

    args = (ro.double().requires_grad_(True), rd.double().requires_grad_(True),
            table0[sel].clone().requires_grad_(True),
            *[w.clone().requires_grad_(True) for w in Ws0])
    assert torch.autograd.gradcheck(fn, args, eps=1e-6, atol=1e-7, rtol=1e-5)


# ---- mutations: what a wrong kernel would produce, applied to the fp32 oracle's gradient ----
def _add_point_grads(g, ref, pts, lvl, corner_w):
    """g[entry] += corner_w[p, k] * dfeat[p, lvl] at the entry of corner k, for p in pts."""
    out = g.clone().view(-1, 2)
    idx = ref['idx'][pts, lvl]                     # [n,8]
    add = corner_w[..., None] * ref['dfeat'][pts, lvl][:, None, :]   # [n,8,2]
    out.index_add_(0, idx.reshape(-1), add.reshape(-1, 2))
    return out.reshape(-1)


def test_mutation_drop_split_pair_corner(step4097):
    """The x+1 corner of split pairs (i1 != i0 ^ 1) lost on one fine hashed level, 1 % of points."""
    _, ref, cand, sdf = step4097
    lvl = 13
    assert bool(ref['layout']['hashed'][lvl])
    pts = torch.arange(0, ref['idx'].shape[0], 100)
    idx = ref['idx'][pts, lvl]
    cw = torch.zeros(len(pts), 8, dtype=torch.float64)
    for k in (0, 2, 4, 6):
        split = idx[:, k + 1] != (idx[:, k] ^ 1)
        cw[:, k + 1] = -ref['wc'][pts, lvl, k + 1] * split
    assert bool((cw != 0).any())
    mut = dict(cand, d_table=_add_point_grads(cand['d_table'], ref, pts, lvl, cw))
    assert _flagged(ref, mut, sdf) == []


def test_mutation_swap_corners_dense_wrap(step4097):
    """Corners k and k + 1 swapped on a dense level for the points outside [0, 1)."""
    _, ref, cand, sdf = step4097
    lvl = 2
    assert not bool(ref['layout']['hashed'][lvl])
    x = ref['x32']
    pts = torch.nonzero(((x < 0) | (x >= 1)).any(1)).reshape(-1)
    assert len(pts) > 100
    wc = ref['wc'][pts, lvl]
    cw = torch.zeros_like(wc)
    for k in (0, 2, 4, 6):
        cw[:, k] = wc[:, k + 1] - wc[:, k]
        cw[:, k + 1] = wc[:, k] - wc[:, k + 1]
    mut = dict(cand, d_table=_add_point_grads(cand['d_table'], ref, pts, lvl, cw))
    assert _flagged(ref, mut, sdf) == []


def test_mutation_scale_level_12(step4097):
    _, ref, cand, sdf = step4097
    a, b = F.level_slices(ref['layout'])[12]
    g = cand['d_table'].clone()
    g[a:b] *= 1.01
    assert _flagged(ref, dict(cand, d_table=g), sdf) == []


@pytest.mark.parametrize('which', ['smallest', 'largest'])
@pytest.mark.parametrize('key', ['d_rays_o', 'd_rays_d'])
def test_mutation_copy_neighbour_ray(step4097, which, key):
    _, ref, cand, sdf = step4097
    mag = ref['grads'][key].norm(dim=1)
    r = int(mag.argmin() if which == 'smallest' else mag.argmax())
    src = r - 1 if r > 0 else r + 1
    g = cand[key].clone()
    g[r] = g[src]
    assert _flagged(ref, dict(cand, **{key: g}), sdf) == []


def test_mutation_drop_last_ray_col1(step4097):
    """R = 4097: the last ray (alone in the final unit) missing from d_w_col1."""
    _, ref, cand, sdf = step4097
    S = ref['S']
    last = slice((ref['R'] - 1) * S, ref['R'] * S)
    contrib = ref['draw'][last, :3].T @ ref['hc'][last]
    assert bool((contrib != 0).any())
    mut = dict(cand, d_w_col1=cand['d_w_col1'] - contrib)
    assert 0 not in _flagged(ref, mut, sdf, modes=(0,))


@pytest.mark.parametrize('sp, voxel', [(3, 0.1), (6, 0.1), (40, 0.15)])
def test_smoothness_replay_lattice_arguments(sp, voxel):
    """smoothness_replay on a lattice other than the config's agrees with the fp32 oracle's
    autograd of the same lattice to fp32 rounding within the entry bound A, and with no
    arguments it replays the config's lattice."""
    ora = _oracle(0.1)
    rnd = torch.tensor([0.3, 0.7, 0.1, 0.9, 0.2, 0.5]).reshape(2, 3)
    loss64, g64, A, _, terms = F.smoothness_replay(ora, rnd, sample_points=sp, voxel=voxel,
                                                   margin=0.05, with_terms=True)
    assert len(terms) == 16 and min(terms) >= 1
    p = ora.smooth_points(rnd, sp, voxel, 0.05)
    assert p.shape == (sp - 1,) * 3 + (3,)
    f = ora.embed_fn(p.reshape(-1, 3)).reshape(*p.shape[:-1], -1)
    tv = sum((torch.diff(f, dim=d) ** 2).sum() for d in range(3)) / sp ** 3
    tv.backward()
    err = (ora.embed_fn.params.grad.double() - g64).abs()
    assert not bool(((A == 0) & (err > 0)).any())
    assert float((err[A > 0] / A[A > 0]).max()) < 1e-5
    assert abs(float(tv.detach()) - float(loss64)) <= 1e-6 * float(loss64)
    c = ora.cfg
    dflt = F.smoothness_replay(ora, rnd)
    expl = F.smoothness_replay(ora, rnd, sample_points=c.smooth_pts, voxel=c.smooth_vox,
                               margin=c.smooth_margin)
    assert all(torch.equal(a, b) for a, b in zip(dflt[:3], expl[:3]))
