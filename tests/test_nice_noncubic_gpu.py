"""NICE-SLAM step on a non-cubic scene, judged per grid entry, per colour-decoder element and
per ray against the fp32 oracle (oracle/nice.py).

The parity tests of test_nice_gpu.py run on the cube [-2, 2]^3, where nx == ny == nz and every
axis has the same bound, and judge each gradient by one relative L2 per tensor.  An axis swap
in the grid shape, the bound or the voxel offset, a corner scattered into the neighbouring
cell, one wrong weight element or a single wrong ray would pass them.  Here the bound gives
pairwise distinct nx, ny, nz for every grid, and the checks are (``report``):

  entry   per grid: max |g - g_o| / max |g_o|                 (one wrong block of cells shows)
  weight  per colour-decoder tensor and element: |g - g_o| / (|g_o| + 1e-2 max |g_o|); row 3 of
          output_linear (the unused fourth output) must be exactly 0 in both
  ray     per ray and component: |g - g_o| / (|g_o|_ray + 1e-2 mean |g_o|_ray)
  fwd     max abs of rgb, depth, uncertainty;  loss: relative per term

The rays in the face planes x = bmin and x = bmax pin the border rule of F.grid_sample
(padding 'border', align_corners=True): the coordinate gradient is zero for ix <= 0 and
ix >= size - 1, equality included.  Their samples have a normalised x of exactly -1 and 1.

Gates (GATES, one set for every case): about 4x the worst value observed on an H100 80GB HBM3
(power limit 400 W), and below the smallest ratio the CPU mutations at the end of this file
produce (each is asserted to fail the gates).  The networks come from nice_pair (seeded, grid
amplitude 30, B scaled by 0.2 except in ref_b_map, where B keeps the reference's std 25 and the
sin() arguments reach hundreds of radians); runs repeat to the last digits of the atomics.

  check    worst observed (case)           gate      smallest mutation ratio (mutation)
  entry    2.9e-5 (last_cell_map)          1.5e-4    0.44   (corner moved to the x-neighbour)
  weight   1.1e-4 (ref_b_map)              5e-4      9.9e-4 (one element scaled by 1 + 1e-3)
  ray      9.7e-5 (ref_b_map)              4e-4      0.95   (largest ray copied from neighbour)
  fwd      3.6e-5 (ref_b_map)              2e-4
  loss     1.2e-6 (middle_trk)             1e-5

The other mutations: upper corner dropped on the last cell 0.54-0.82 (entry), middle grid fed
through the fine decoder's feature 0.65 (entry), upper median in tracking 49 (ray), the one-sided
border derivative on the face-plane rays 1.0 (ray).  On the GPU the face-plane rays stay within
2.1e-5; with the one-sided derivative src_index had before the border fix they gave 1.5
(mapping) and 2.3 (tracking).
"""
import contextlib

import numpy as np
import pytest
import torch

from helpers import max_abs
from test_nice_gpu import nice_pair

BOUND_NC = np.array([[-2.0, 2.4], [-1.5, 2.2], [-2.3, 1.6]])
SHAPES_NC = {'grid_middle': (12, 11, 14), 'grid_fine': (25, 23, 28),
             'grid_color': (25, 23, 28), 'grid_coarse': (4, 3, 4)}
GATES = dict(entry=1.5e-4, weight=5e-4, ray=4e-4, fwd=2e-4, loss=1e-5)
GRIDS = ('grid_middle', 'grid_fine', 'grid_color', 'grid_coarse')


def test_noncubic_grid_shapes():
    """(Z, Y, X) of every grid on the non-cubic bound: nx, ny, nz pairwise distinct for
    middle, fine and colour; the coarse grid is not a cube; model and oracle agree."""
    ora, model = nice_pair('cpu', bound=BOUND_NC, coarse=True)
    for k, shp in SHAPES_NC.items():
        assert tuple(ora.grids[k].shape[2:]) == shp, k
        assert tuple(model.grids[k].shape[:3]) == shp, k
        if k != 'grid_coarse':
            assert len(set(shp)) == 3, k
    assert len(set(SHAPES_NC['grid_coarse'])) > 1


# ------------------------------------------------------------------ batches ---
def _rays(name):
    """(rays_o, rays_d, target_s, target_d) of a named batch."""
    R = {'one': 1, 'two': 2, 'odd': 333, 'outside': 400, 'zero_depth': 200}.get(
        name, 1000 if name == 'default' else 200)
    g = torch.Generator().manual_seed(R + len(name))
    lo = torch.tensor(BOUND_NC[:, 0], dtype=torch.float32)
    ext = torch.tensor(BOUND_NC[:, 1] - BOUND_NC[:, 0], dtype=torch.float32)
    ro = lo + ext * (0.3 + 0.4 * torch.rand(R, 3, generator=g))
    rd = torch.nn.functional.normalize(torch.randn(R, 3, generator=g), dim=-1)
    td = torch.rand(R, 1, generator=g) * 1.5 + 0.3
    td[3::7] = 0
    ts = torch.rand(R, 3, generator=g)
    if name == 'outside':     # far samples leave the bound through all six faces
        td = td * 4 + 1.0
        td[3::7] = 0
    if name == 'zero_depth':
        td[::3] = 0
    if name == 'all_zero':    # every target depth 0: all samples within 1 mm of the origin
        td.zero_()
    if name == 'tracking':    # duplicated rays (median ties) and a few outlier depths
        ro[100:150], rd[100:150], td[100:150] = ro[:50], rd[:50], td[:50]
        ts[100:150] = ts[:50]
        td[5::40] = 6.0
    if name == 'two':         # one outlier: the lower and the upper median differ by far
        td[1] = td[0] * 30
    if name == 'last_cell':   # rays starting inside the last cell of each axis of the fine grids
        from oracle.nice import load_bound
        bmax = load_bound(BOUND_NC)[:, 1]
        for a in range(3):
            ro[a::3, a] = float(bmax[a]) - 0.08
    return ro, rd, ts, td


def face_rays():
    """48 rays in the planes x = bmin and x = bmax of the bound (as load_bound left it: both
    fp32-representable), so that every sample has a normalised x of exactly -1 or 1, followed
    by 16 ordinary rays.  Returns the batch and the [R] mask of face rays."""
    from oracle.nice import load_bound
    bb = load_bound(BOUND_NC)
    bmin, bmax = float(bb[0, 0]), float(bb[0, 1])
    assert float(np.float32(bmin)) == bmin and float(np.float32(bmax)) == bmax
    ro, rd, ts, td = _rays('faces')
    R, nf = 64, 48
    ro, rd, ts, td = ro[:R].clone(), rd[:R].clone(), ts[:R], td[:R].clone()
    td[:] = td.clamp_min(0.3)
    ro[:nf // 2, 0], ro[nf // 2:nf, 0] = bmin, bmax
    rd[:nf, 0] = 0
    rd = torch.nn.functional.normalize(rd, dim=-1)
    assert bool((rd[:nf, 0] == 0).all())
    face = torch.zeros(R, dtype=torch.bool)
    face[:nf] = True
    return (ro, rd, ts, td), face


def kernel_sample_z(ora, ro, rd, td):
    """ora.sample_z with the kernel's far_bb: for a ray in a face plane (bound - o) / d is 0/0,
    which torch.max turns into NaN and the kernel's fmax drops."""
    orig = torch.max

    def fmax(t, *a, **k):
        if a == (2,) or k.get('dim') == 2:
            t = torch.nan_to_num(t, nan=-float('inf'))
        return orig(t, *a, **k)
    torch.max = fmax
    try:
        return ora.sample_z(ro, rd, td)
    finally:
        torch.max = orig


# ------------------------------------------------------------------- steps ---
def oracle_step(ora, stage, is_mapping, ro, rd, ts, td, z=None):
    """fp32 oracle step -> gradients and outputs in the layout ``report`` takes (grids
    channel-last [Z,Y,X,C], colour tensors in ConvOnet's MLP.tensors() order)."""
    for p in ora.parameters():
        p.grad = None
    if z is not None:
        ora.sample_z = lambda *a: z
    ro = ro.detach().clone().requires_grad_(True)
    rd = rd.detach().clone().requires_grad_(True)
    out, ld, tot = ora.step(ro, rd, ts, td, is_mapping, stage)
    tot.backward()
    if z is not None:
        del ora.sample_z
    c = ora.color
    col = [c.B]
    for i in range(5):
        col += [c.pts[i].weight, c.pts[i].bias]
    for i in range(5):
        col += [c.fc_c[i].weight, c.fc_c[i].bias]
    col += [c.out.weight, c.out.bias]
    return dict(grids={k: ora.grids[k].grad.squeeze(0).permute(1, 2, 3, 0)
                       for k in GRIDS if k in ora.grids and ora.grids[k].grad is not None},
                color=[t.grad for t in col] if stage == 'color' else None,
                d_rays_o=ro.grad, d_rays_d=rd.grad,
                fwd={k: out[k].detach() for k in ('rgb', 'depth', 'uncertainty')},
                losses={k: float(v.detach()) for k, v in ld.items()}, z=out['z_vals'])


def model_step(model, stage, is_mapping, ro, rd, ts, td, dev):
    S = 32 if stage == 'coarse' else 48
    z = torch.empty(ro.shape[0], S, dtype=torch.float64, device=dev)
    model._z_capture = z
    rk = ro.detach().to(dev).requires_grad_(True)
    dk = rd.detach().to(dev).requires_grad_(True)
    inp = dict(rays_o=rk, rays_d=dk, target_s=ts.to(dev), target_d=td.to(dev), stage=stage,
               is_mapping=is_mapping)
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


def report(ref, cand, rays=None):
    """Ratios of a candidate step against the oracle's (see the module docstring); ``rays``
    [R] bool restricts the ray check."""
    f64 = lambda t: t.detach().cpu().double()
    rep = dict(entry={}, weight={}, ray={})
    assert set(cand['grids']) == set(ref['grids'])
    for k, go in ref['grids'].items():
        go, g = f64(go), f64(cand['grids'][k])
        rep['entry'][k] = float((g - go).abs().max() / go.abs().max().clamp_min(1e-30))
    if ref['color'] is not None:
        for i, (g, go) in enumerate(zip(cand['color'], ref['color'])):
            g, go = f64(g), f64(go)
            if i in (21, 22):   # output_linear: row 3 takes no gradient, exactly
                assert float(g[3].abs().max()) == 0.0 and float(go[3].abs().max()) == 0.0
            den = go.abs() + 1e-2 * go.abs().max()
            rep['weight'][i] = float(((g - go).abs() / den.clamp_min(1e-30)).max())
    for key in ('d_rays_o', 'd_rays_d'):
        g, go = f64(cand[key]), f64(ref[key])
        if rays is not None:
            g, go = g[rays], go[rays]
        den = go.abs().amax(1, keepdim=True) + 1e-2 * go.abs().amax(1).mean()
        rep['ray'][key] = float(((g - go).abs() / den.clamp_min(1e-30)).max())
    rep['fwd'] = max(max_abs(cand['fwd'][k], ref['fwd'][k]) for k in ref['fwd'])
    assert set(cand['losses']) == set(ref['losses'])
    rep['loss'] = max(abs(cand['losses'][k] - v) / max(abs(v), 1.0)
                      for k, v in ref['losses'].items())
    return rep


def failures(rep, gates):
    out = [f'entry {k}: {v:.3g}' for k, v in rep['entry'].items() if not v <= gates['entry']]
    out += [f'weight {k}: {v:.3g}' for k, v in rep['weight'].items() if not v <= gates['weight']]
    out += [f'ray {k}: {v:.3g}' for k, v in rep['ray'].items() if not v <= gates['ray']]
    out += [f'{k}: {rep[k]:.3g}' for k in ('fwd', 'loss') if not rep[k] <= gates[k]]
    return out


# --------------------------------------------------------------- GPU cases ---
CASES = {
    # name: (stage, is_mapping, rays, B scale)
    'color_map': ('color', True, 'default', 0.2),
    'color_trk': ('color', False, 'tracking', 0.2),
    'middle_map': ('middle', True, 'odd', 0.2),
    'middle_trk': ('middle', False, 'odd', 0.2),
    'fine_map': ('fine', True, 'odd', 0.2),
    'fine_trk': ('fine', False, 'odd', 0.2),
    'coarse_map': ('coarse', True, 'odd', 0.2),   # the coarse stage only maps
    'one_map': ('color', True, 'one', 0.2),
    'one_trk': ('color', False, 'one', 0.2),
    'two_trk': ('color', False, 'two', 0.2),
    'outside_map': ('color', True, 'outside', 0.2),
    'last_cell_map': ('color', True, 'last_cell', 0.2),
    'zero_depth_map': ('color', True, 'zero_depth', 0.2),
    'zero_depth_trk': ('color', False, 'zero_depth', 0.2),
    'all_zero_map': ('color', True, 'all_zero', 0.2),
    'ref_b_map': ('color', True, 'default', 1.0),  # B at the reference's init (std 25)
}


def case_report(dev, name):
    stage, is_mapping, rays, b = CASES[name]
    ro, rd, ts, td = _rays(rays)
    ora, model = nice_pair(dev, bound=BOUND_NC, coarse=stage == 'coarse', b_scale=b)
    cand = model_step(model, stage, is_mapping, ro, rd, ts, td, dev)
    ref = oracle_step(ora, stage, is_mapping, ro, rd, ts, td)
    assert torch.equal(cand['z'], ref['z'])                    # f64 sample depths: bit-exact
    return report(ref, cand)


def face_report(dev, is_mapping):
    (ro, rd, ts, td), face = face_rays()
    ora, model = nice_pair(dev, bound=BOUND_NC)
    cand = model_step(model, 'color', is_mapping, ro, rd, ts, td, dev)
    z = kernel_sample_z(ora, ro, rd, td)
    assert torch.equal(cand['z'], z)            # every ray, with the kernel's fmax far_bb
    z_o = ora.sample_z(ro, rd, td)
    assert torch.equal(cand['z'][~face], z_o[~face])            # torch's own rule elsewhere
    ref = oracle_step(ora, 'color', is_mapping, ro, rd, ts, td, z=z)
    return report(ref, cand, rays=face), report(ref, cand, rays=~face)


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(CASES))
def test_noncubic_step_vs_oracle(cuda_dev, name):
    rep = case_report(cuda_dev, name)
    bad = failures(rep, GATES)
    assert not bad, (name, bad, rep)


@pytest.mark.gpu
@pytest.mark.parametrize('is_mapping', [True, False])
def test_face_plane_rays_border_rule(cuda_dev, is_mapping):
    """Rays in the planes x = bmin (ix == 0) and x = bmax (ix == size - 1): torch's
    grid_sample gives the x coordinate zero gradient there; a one-sided derivative, or the
    lower corner alone at the upper face, moves d_rays_o / d_rays_d by a large fraction."""
    for rep in face_report(cuda_dev, is_mapping):
        bad = failures(rep, GATES)
        assert not bad, (bad, rep)


@pytest.mark.gpu
def test_tracking_median_guard(cuda_dev):
    """Tracking takes the batch median in one block: 8192 rays are accepted, 8193 refused."""
    from xrdslam_b200._cabi import XrdError
    _, model = nice_pair(cuda_dev, bound=BOUND_NC)
    for R, ok in ((8192, True), (8193, False)):
        g = torch.Generator().manual_seed(R)
        ro = torch.rand(R, 3, generator=g).to(cuda_dev)
        rd = torch.nn.functional.normalize(torch.randn(R, 3, generator=g), dim=-1).to(cuda_dev)
        td = (torch.rand(R, 1, generator=g) + 0.3).to(cuda_dev)
        ts = torch.rand(R, 3, generator=g).to(cuda_dev)
        if ok:
            out, grads = model._launch('color', False, ro, rd, ts, td, True, need_rays=True)
            torch.cuda.synchronize()
            assert bool(torch.isfinite(grads['d_rays_o']).all())
        else:
            with pytest.raises(XrdError):
                model._launch('color', False, ro, rd, ts, td, True, need_rays=True)


# ------------------------------------------------- CPU: mutations are flagged ---
# What a wrong kernel would produce, applied to the oracle's own gradient: each must fail the
# gates above, so the gates are below the size of every such fault.
def _step_with_features(ora, stage, is_mapping, batch, z=None):
    """oracle_step that also returns, per call of sample_grid on the colour grid, the points
    and d loss / d feature [P, 32]."""
    import oracle.nice as N
    rec = []
    orig = N.sample_grid

    def sample(p, grid, bound):
        c = orig(p, grid, bound)
        if grid is ora.grids['grid_color'] and c.requires_grad:
            c.retain_grad()
            rec.append((p.detach(), c, bound))
        return c
    N.sample_grid = sample
    try:
        ref = oracle_step(ora, stage, is_mapping, *batch, z=z)
    finally:
        N.sample_grid = orig
    (p, c, bound), = rec
    return ref, p, c.grad.detach(), bound


def _cells(p, bound, grid_shape):
    """grid_sample's cell of each point (fp32, border clip): i0 [P,3] (x,y,z), f [P,3]."""
    Z, Y, X = grid_shape
    xn = torch.stack([((p[:, d] - bound[d, 0]) / (bound[d, 1] - bound[d, 0])) * 2 - 1.0
                      for d in range(3)], 1).float()
    i0, f = [], []
    for d, n in enumerate((X, Y, Z)):
        ix = (((xn[:, d] + 1) / 2) * (n - 1)).clamp(0, n - 1)
        i0.append(torch.floor(ix).long())
        f.append(ix - torch.floor(ix))
    return torch.stack(i0, 1), torch.stack(f, 1).double(), xn


@pytest.fixture(scope='module')
def color_step():
    ora, _ = nice_pair('cpu', bound=BOUND_NC)
    batch = _rays('last_cell')
    ref, p, dc, bound = _step_with_features(ora, 'color', True, batch)
    return ora, batch, ref, p, dc.double(), bound


def _flagged(ref, cand, rays=None):
    return failures(report(ref, cand, rays), GATES)


def _with_grid(ref, key, g):
    return dict(ref, grids=dict(ref['grids'], **{key: g}))


def _scatter(g, idx_zyx, val):
    g = g.clone().double()
    g.index_put_(tuple(idx_zyx.T), val, accumulate=True)
    return g


def test_mutation_corner_moved_to_x_neighbour(color_step):
    """Corner (0,0,0) of every 10th point scattered into the x-neighbour voxel."""
    ora, _, ref, p, dc, bound = color_step
    shp = tuple(ora.grids['grid_color'].shape[2:])
    i0, f, _ = _cells(p, bound, shp)
    sel = torch.arange(0, p.shape[0], 10)
    sel = sel[(i0[sel, 0] < shp[2] - 1) & (dc[sel].abs().sum(1) > 0)]
    assert len(sel) > 100
    w = ((1 - f[sel, 0]) * (1 - f[sel, 1]) * (1 - f[sel, 2]))[:, None] * dc[sel]
    zyx = i0[sel].flip(1)
    g = _scatter(ref['grids']['grid_color'], zyx, -w)
    g = _scatter(g, zyx + torch.tensor([0, 0, 1]), w)
    assert any('grid_color' in m for m in _flagged(ref, _with_grid(ref, 'grid_color', g)))


@pytest.mark.parametrize('axis', [0, 1, 2])
def test_mutation_upper_corner_dropped_on_last_cell(color_step, axis):
    """The upper-corner contributions along one axis lost for points in its last cell."""
    ora, _, ref, p, dc, bound = color_step
    shp = tuple(ora.grids['grid_color'].shape[2:])
    n = shp[::-1][axis]
    i0, f, xn = _cells(p, bound, shp)
    sel = torch.nonzero((i0[:, axis] == n - 2) & (xn.abs() < 1).all(1)).reshape(-1)
    assert len(sel) > 0
    g = ref['grids']['grid_color']
    for k in range(8):
        o = torch.tensor([(k >> d) & 1 for d in range(3)])
        if not o[axis]:
            continue
        w = torch.ones(len(sel), dtype=torch.float64)
        for d in range(3):
            w = w * (f[sel, d] if o[d] else 1 - f[sel, d])
        g = _scatter(g, (i0[sel] + o).flip(1), -(w[:, None] * dc[sel]))
    assert any('grid_color' in m for m in _flagged(ref, _with_grid(ref, 'grid_color', g)))


@pytest.mark.parametrize('tensor', [1, 7, 11, 21])   # pts0.w, pts3.w, fcc0.w, output_linear.w
def test_mutation_weight_element_scaled(color_step, tensor):
    """The largest element of one colour-decoder weight gradient scaled by 1 + 1e-3."""
    _, _, ref, *_ = color_step
    col = [t.clone() for t in ref['color']]
    flat = col[tensor].view(-1)
    flat[flat.abs().argmax()] *= 1 + 1e-3
    assert f'weight {tensor}: ' in ' '.join(_flagged(ref, dict(ref, color=col)))


@pytest.mark.parametrize('which', ['smallest', 'largest'])
@pytest.mark.parametrize('key', ['d_rays_o', 'd_rays_d'])
def test_mutation_ray_copied_from_neighbour(color_step, key, which):
    _, _, ref, *_ = color_step
    mag = ref[key].norm(dim=1)
    r = int(mag.argmin() if which == 'smallest' else mag.argmax())
    g = ref[key].clone()
    g[r] = g[r - 1 if r > 0 else r + 1]
    assert any(key in m for m in _flagged(ref, dict(ref, **{key: g})))


def test_mutation_one_sided_border_derivative():
    """src_index before the border fix: the x coordinate kept its gradient at ix == 0 (the
    right-sided derivative) and at ix == size - 1 (the lower corner alone, -v_hi * mult)."""
    ora, _ = nice_pair('cpu', bound=BOUND_NC)
    batch, face = face_rays()
    z = kernel_sample_z(ora, *batch[:2], batch[3])
    ref, p, dc, bound = _step_with_features(ora, 'color', True, batch, z=z)
    dc = dc.double()
    grid = ora.grids['grid_color'].detach().squeeze(0).permute(1, 2, 3, 0).double()
    Z, Y, X = grid.shape[:3]
    i0, f, xn = _cells(p, bound, (Z, Y, X))
    on = (xn[:, 0].abs() == 1) & (dc.abs().sum(1) > 0)
    assert int(on.sum()) >= 40
    gx = torch.zeros(p.shape[0], dtype=torch.float64)
    for k in range(4):                      # (dy, dz) corners
        dy, dz = k & 1, k >> 1
        y, zz = (i0[:, 1] + dy).clamp(max=Y - 1), (i0[:, 2] + dz).clamp(max=Z - 1)
        w = (f[:, 1] if dy else 1 - f[:, 1]) * (f[:, 2] if dz else 1 - f[:, 2])
        w = w * (i0[:, 1] + dy < Y) * (i0[:, 2] + dz < Z)
        x0 = i0[:, 0]
        lo = (grid[zz, y, x0] * dc).sum(1)
        hi = (grid[zz, y, (x0 + 1).clamp(max=X - 1)] * dc).sum(1) * (x0 + 1 < X)
        gx = gx + w * (hi - lo)
    dpx = gx * on * (X - 1) / 2 * 2 / float(bound[0, 1] - bound[0, 0])
    R = face.shape[0]
    dpx = dpx.reshape(R, -1)
    ro, rd = ref['d_rays_o'].clone(), ref['d_rays_d'].clone()
    ro[:, 0] += dpx.sum(1).float()
    rd[:, 0] += (dpx * z).sum(1).float()
    bad = _flagged(ref, dict(ref, d_rays_o=ro, d_rays_d=rd), rays=face)
    assert any('d_rays_o' in m for m in bad) and any('d_rays_d' in m for m in bad)


def test_mutation_middle_grid_through_fine_feature():
    """The middle grid taking gradient through the fine decoder's concatenated feature, which
    the reference samples under no_grad."""
    ora, _ = nice_pair('cpu', bound=BOUND_NC)
    batch = _rays('odd')
    ref = oracle_step(ora, 'fine', True, *batch)
    orig = torch.no_grad
    torch.no_grad = contextlib.nullcontext
    try:
        mut = oracle_step(ora, 'fine', True, *batch)
    finally:
        torch.no_grad = orig
    assert any('grid_middle' in m for m in _flagged(ref, mut))


def test_mutation_upper_median_in_tracking():
    """Tracking masks rays with |D - d| / sqrt(var) >= 10 median: the upper median of an even
    batch (torch.median returns the lower one) keeps the outlier ray of this batch live."""
    ora, _ = nice_pair('cpu', bound=BOUND_NC)
    batch = _rays('two')
    ref = oracle_step(ora, 'color', False, *batch)
    orig = torch.Tensor.median
    torch.Tensor.median = lambda t, *a, **k: \
        t.sort()[0][t.numel() // 2] if not a and not k else orig(t, *a, **k)
    try:
        mut = oracle_step(ora, 'color', False, *batch)
    finally:
        torch.Tensor.median = orig
    bad = _flagged(ref, mut)
    assert any('d_rays' in m for m in bad) and any('loss' in m for m in bad)
