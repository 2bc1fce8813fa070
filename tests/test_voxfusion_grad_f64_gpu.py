"""Vox-Fusion render-and-optimise step (xrd_voxfusion_render, all four GEMM arithmetic modes)
against the float64 replay of oracle/voxfusion_f64.py: every embedding entry, every element of
the ten decoder gradients, every ray and component, every loss term and the rendered colour and
depth.  The whole-tensor relative L2 of test_voxfusion_gpu.py lets a lost staging tail of the
weight-gradient kernel, a wrong corner of one voxel or a wrong ray through; these checks do not.

Gates (per GEMM mode): about 4x the worst ratio over all cases below, and below the smallest
ratio the mutations of test_voxfusion_f64_reference_cpu.py produce at that check:

  mode  check   worst on the H100 (case)     gate     mutation floor (CPU)
  0     entry   1.3e-8  (p_small)            6e-8     7.1e-5  corner 0 -> vid[4], one voxel
        weight  1.7e-7  (p_small)            5e-7     9.9e-7  wc1 element x (1 + 1e-3)
        ray     1.3e-9  (depth_edges)        5e-9     3.0e-5  d_rays_d without z, one ray
        loss    5.9e-6  (depth_edges)        2.4e-5
        fwd     7.9e-7                       3.2e-6
  1, 3  entry   1.6e-7  (depth_edges)        6e-7     7.1e-5  as above
        weight  2.2e-6  (p_large)            9e-6     2.3e-4  w1 element x (1 + 1e-3);
                                                      3.8e-4  last 64 points of w0 / b0
        ray     1.7e-8  (depth_edges)        7e-8     3.0e-5  as above
        loss    5.9e-6  (depth_edges)        2.4e-5
        fwd     1.0e-6                       4e-6
  2     weight  1.8e-3  (depth_edges)        7e-3     8.2e-3  last 64 points of wc0 / bc0
        loss    2.3e-4  (depth_edges)        1e-3
        fwd     7.0e-4                       3e-3
  Plain TF32 (mode 2) has a 2e-3 ambiguity threshold: about 93 % of the points then hold an
  ambiguous unit, so the entry and ray checks of mode 2 exempt nearly everything (observed 0).
  Rays with another step: 0 in modes 0, 1, 3; mode 2 up to 2 of 5115, 90 of 5115 in no_sign.
  Other floors: axis weight from another axis 2.1e-4 (entry), wc0 columns 128..143 zero 0.87,
  zlim one sample later 1.0e-3 (weight), per-ray Q3 normaliser 0.51 (weight), neighbour ray
  copied 5.6e-5 (ray), last 64 points of w1 / ws / wc1: 2.3e-3 / 1.5e-3 / 1.1e-2 (weight).
  A 1e-3 change of the most exposed element of w0, ws and wc1 (6.4e-6, 2.5e-6, 1e-6) stays
  under the weight gate of modes 1 and 3; the fp32 gate of mode 0 flags it.
  Measured on one H100 80GB HBM3 at a 400 W power limit; the file runs in about 14 s there.

The fp32 CPU oracle itself stays within entry 4e-9, weight 2.4e-7, ray 1.1e-10, loss 1.1e-7 and
forward 2.6e-7 of float64 on the CPU oracle case.
"""
import contextlib

import pytest
import torch

pytestmark = pytest.mark.gpu

# ReLU ambiguity threshold |pre| / sum|terms| for the candidate's forward arithmetic:
# fp32 SIMT (0) and 3xTF32 (1, 3) round like fp32, plain TF32 (2) has a 10-bit mantissa
AMB = {0: 1e-5, 1: 1e-5, 2: 2e-3, 3: 1e-5}
GATES = {
    0: dict(entry=6e-8, weight=5e-7, ray=5e-9, loss=2.4e-5, fwd=3.2e-6),
    1: dict(entry=6e-7, weight=9e-6, ray=7e-8, loss=2.4e-5, fwd=4e-6),
    2: dict(entry=6e-7, weight=7e-3, ray=7e-8, loss=1e-3, fwd=3e-3),
    3: dict(entry=6e-7, weight=9e-6, ray=7e-8, loss=2.4e-5, fwd=4e-6),
}
MODES = (0, 1, 2, 3)
# at most Rh / FLIP_DIV rays may take another step; plain TF32 moves the sign change of the
# lifted-sdf batch (many samples near sdf 0) on 90 of 5115 rays
FLIP_DIV = {0: 200, 1: 200, 2: 50, 3: 200}
N_SCENE = 8192          # rays of the scene batch the cases are cut from
BENCH_R = 5 * 1024      # bench_workloads.VoxWorkload: 5 keyframes x 1024 rays
MISS_O, MISS_D = (1.0, 1.0, 1.0), (0.0, 0.0, 1.0)
CASES = ('bench', 'p_small', 'p_tail', 'p_large', 'one', 'long', 'depth_edges', 'no_sign')


@contextlib.contextmanager
def gemm_mode(mode):
    from xrdslam_b200 import _cabi
    lib = _cabi.lib()
    _cabi.check('xrd_debug_gemm_mode', lib.xrd_debug_gemm_mode(mode))
    try:
        yield
    finally:
        lib.xrd_debug_gemm_mode(1)


def _dec(model):
    return [t.detach() for t in model.decoder.tensors()]


class _Refs:
    """One map (the scene of test_voxfusion_gpu, embeddings randn * 0.3), the case batches cut
    from its rays, and their float64 replays, each computed once."""

    def __init__(self, dev):
        from test_voxfusion_gpu import scene
        self.dev = dev
        model, ro, rd, ts, td = scene(dev, R=N_SCENE, seed=4)
        with torch.no_grad():
            g = torch.Generator().manual_seed(9)
            model.embeddings.copy_(torch.randn(model.embeddings.shape, generator=g) * 0.3)
        g = torch.Generator().manual_seed(5)
        noise = torch.rand(N_SCENE, model.config.max_samples_per_ray, generator=g)
        self.model = model
        self.rays = [t.to(dev) for t in (ro, rd, ts, td, noise.clamp(0.001, 0.999))]
        self.cache = {}

    def march(self, rays):
        m = self.model.march(rays[0], rays[1], rays[4])
        return m

    def prefix(self, n):
        return [t[:n] for t in self.rays]

    def _search(self, ok, lo, hi):
        """Smallest prefix length n in [lo, hi] with ok(n_points of the prefix)."""
        while lo < hi:
            mid = (lo + hi) // 2
            if ok(self.march(self.prefix(mid))['n_points']):
                hi = mid
            else:
                lo = mid + 1
        return lo

    def batch(self, name):
        """(rays_o, rays_d, target_s, target_d, noise) of a case."""
        if name in ('bench', 'no_sign'):
            return self.prefix(BENCH_R)
        if name == 'p_small':     # the whole chain on k_gemm_tc / k_gemm: P < 512
            n = self._search(lambda P: P >= 512, 1, 64) - 1
            return self.prefix(n)
        if name == 'p_tail':      # t5 128-point tile tail and k_dw_tc 64-point staging tail
            n = self._search(lambda P: P >= 1500, 1, 256)
            while self.march(self.prefix(n))['n_points'] % 64 == 0:
                n += 1
            return self.prefix(n)
        if name == 'p_large':     # the whole scene batch: well past 2^17 points
            return self.rays
        if name == 'one':
            m = self.march(self.prefix(64))
            r = int(torch.nonzero(m['smp_count'] > 16)[0])
            return [t[r:r + 1] for t in self.rays]
        if name == 'long':        # rays of more than 64 samples, of 33..64 and of at most 32
            m = self.march(self.rays)
            cnt = m['smp_count']
            sel = torch.cat([torch.nonzero(cnt > 64).reshape(-1)[:96],
                             torch.nonzero((cnt > 32) & (cnt <= 64)).reshape(-1)[:64],
                             torch.nonzero((cnt > 0) & (cnt <= 32)).reshape(-1)[:64]])
            sel = sel[torch.randperm(sel.numel(), generator=torch.Generator().manual_seed(1))
                      .to(sel.device)]
            return [t[sel] for t in self.rays]
        if name == 'depth_edges':  # td 0, (0, 0.01], max_dpeth and beyond; misses in between
            ro, rd, ts, td, noise = (t.clone() for t in self.prefix(1024))
            ro[1::2] = torch.tensor(MISS_O, device=self.dev)
            rd[1::2] = torch.tensor(MISS_D, device=self.dev)
            edges = torch.tensor([0.0, 0.004, 0.01, 10.0, 11.5], device=self.dev)
            td[0:400:2, 0] = edges.repeat(40)
            return [ro, rd, ts, td, noise]
        raise KeyError(name)

    def get(self, name):
        if name not in self.cache:
            from oracle import voxfusion_f64 as F
            rays = self.batch(name)
            model = self.model
            dec = _dec(model)
            if name == 'no_sign':  # lift the sdf until about half of the rays stay positive
                ref0 = self.get('bench')['ref']
                sdf, vm = ref0['sdf'], ref0['ctx']['vmask']
                lift = float(torch.quantile(-torch.where(vm, sdf, torch.inf).amin(1), 0.5))
                dec[5] = dec[5].clone()
                dec[5][0] += lift + 1e-3
            m = self.march(rays)
            assert m['overflow'] == 0
            sampled = F.from_march(m)
            ms = model.map_states
            ctx = F.prepare(rays[0], rays[1], rays[2], rays[3], sampled, ms['voxel_center_xyz'],
                            ms['voxel_vertex_idx'], device=self.dev)
            ref = F.replay_step(ctx, model.embeddings, dec)
            self.cache[name] = dict(rays=rays, ref=ref, dec=dec, m=m,
                                    sampled=[t.clone() for t in sampled])
        return self.cache[name]


@pytest.fixture(scope='module')
def refs(cuda_dev):
    return _Refs(cuda_dev)


@contextlib.contextmanager
def _decoder(model, dec):
    """The model's decoder tensors replaced by ``dec`` for the duration of one case."""
    ts = model.decoder.tensors()
    old = [t.detach().clone() for t in ts]
    with torch.no_grad():
        for t, v in zip(ts, dec):
            t.copy_(v)
    try:
        yield
    finally:
        with torch.no_grad():
            for t, v in zip(ts, old):
                t.copy_(v)


def query_sdf(model, ctx, m, rays):
    """The candidate's own per-sample sdf and colour, in the replay's (ray, k) order: the
    render's point order base[r] + k through xrd_voxfusion_query's point mode, which runs the
    render's corners_at and decoder GEMM chain on the same P."""
    from xrdslam_b200 import _cabi
    dev, P = ctx['dev'], ctx['P']
    hit_rows = torch.nonzero(ctx['ray_mask']).reshape(-1)
    r_full = hit_rows[ctx['ray_of']]
    pos = m['smp_base'][r_full].long() + ctx['k_of']
    assert torch.equal(torch.sort(pos).values, torch.arange(P, device=dev))
    z = ctx['z32'][ctx['ray_of'], ctx['k_of']]
    ro, rd = rays[0], rays[1]
    vox = torch.empty(P, dtype=torch.int32, device=dev)
    pts = torch.empty(P, 3, device=dev)
    vox[pos] = ctx['vox'].int()
    pts[pos] = ro[r_full] + rd[r_full] * z[:, None]
    sdf = torch.empty(P, device=dev)
    rgb = torch.empty(P, 3, device=dev)
    ws = torch.empty(_cabi.lib().xrd_voxfusion_query_workspace_bytes(P), dtype=torch.uint8,
                     device=dev)
    model._query(P, vox, xyz=pts, sdf=sdf, rgb=rgb, ws=ws)
    return sdf[pos], rgb[pos]


def composite32(ctx, sdf_p, rgb_p):
    """sdf2weights + composite in fp32 from per-point sdf / colour -> (rgb [Rh,3], depth [Rh])."""
    from oracle import voxfusion_f64 as F
    sdf = F.candidate_sdf(ctx, sdf_p)
    Rh, S = ctx['Rh'], ctx['S']
    col = torch.zeros(Rh * S, 3, device=ctx['dev'])
    col[ctx['flat']] = rgb_p
    tm = F.trunc_mask(ctx, F.sdf_first(sdf)).float()
    a = torch.sigmoid(sdf / ctx['tr']) * torch.sigmoid(-sdf / ctx['tr']) * tm
    w = a / (a.sum(-1, keepdim=True) + 1e-8)
    return (w[..., None] * col.view(Rh, S, 3)).sum(1), (w * ctx['z32']).sum(-1)


def run_case(refs, name, mode, need_rays=True, need_map=True):
    """One step through SparseVoxel._launch under GEMM mode ``mode`` -> (compare report, case)."""
    from oracle import voxfusion_f64 as F
    c = refs.get(name)
    model, ref = refs.model, c['ref']
    ctx = ref['ctx']
    ro, rd, ts, td, noise = c['rays']
    with gemm_mode(mode), _decoder(model, c['dec']):
        out, g = model._launch(ro, rd, ts, td, noise, True, need_rays, need_map)
        sdf_p, rgb_p = query_sdf(model, ctx, model.last_march, c['rays'])
        torch.cuda.synchronize()
    m = model.last_march
    assert m['overflow'] == 0
    # the replay's fp32 inputs: the same march (only the point order base[r] may differ)
    assert m['s_max'] == ctx['S'] and m['n_points'] == ctx['P'] and m['n_hit_rays'] == ctx['Rh']
    for a, b in zip(F.from_march(m), c['sampled']):
        assert torch.equal(a, b)
    for k, v in list(g.items()):
        for t in (v if isinstance(v, list) else [v]):
            if t is not None:
                assert bool(torch.isfinite(t).all()), k
    hm = ctx['ray_mask']
    # the query reproduces the render's sdf and colour: its composite is the render's output
    rgb32, depth32 = composite32(ctx, sdf_p, rgb_p)
    q_err = (float((rgb32 - out['rgb'][hm]).abs().max()),
             float((depth32 - out['depth'][hm]).abs().max()))
    if need_map:
        vid = ctx['vid'].reshape(-1)
        untouched = torch.ones(g['d_emb'].shape[0], dtype=torch.bool, device=refs.dev)
        untouched[vid] = False
        assert bool((g['d_emb'][untouched] == 0).all())
    cand = dict(d_emb=g['d_emb'], d_dec=g['d_dec'], d_rays_o=g['d_rays_o'],
                d_rays_d=g['d_rays_d'], losses=out['losses'], rgb=out['rgb'], depth=out['depth'])
    rep = F.compare(ref, cand, AMB[mode], F.candidate_sdf(ctx, sdf_p))
    return rep, c, g, q_err


QUERY_TOL = (2e-6, 4e-6)   # rgb, depth [m]: the query's composite against the render's output


def _check(rep, c, q_err, mode, name):
    from oracle import voxfusion_f64 as F
    assert q_err[0] < QUERY_TOL[0] and q_err[1] < QUERY_TOL[1], q_err
    # a handful of rays may take another step (sign change or L1 residual sign); they are left
    # out, not the batch
    Rh = c['ref']['ctx']['Rh']
    assert rep['n_flip_rays'] <= max(2, Rh // FLIP_DIV[mode]), rep['n_flip_rays']
    bad = F.failures(rep, GATES[mode])
    assert not bad, (name, mode, bad)


def _case_property(name, c):
    """The property the case claims, checked on its march and batch."""
    ctx = c['ref']['ctx']
    P, cnt = ctx['P'], ctx['count']
    if name == 'bench':
        assert ctx['R'] == BENCH_R
    elif name == 'p_small':
        assert 0 < P < 512
    elif name == 'p_tail':
        assert P >= 512 and P % 64 != 0
    elif name == 'p_large':
        assert P > 1 << 17
    elif name == 'one':
        assert ctx['R'] == 1 and ctx['Rh'] == 1
    elif name == 'long':
        assert bool((cnt > 64).any()) and bool(((cnt > 32) & (cnt <= 64)).any())
        assert bool((cnt < ctx['S']).any())
    elif name == 'depth_edges':
        td = ctx['td32']
        assert bool((td == 0).any()) and bool(((td > 0) & (td <= 0.01)).any())
        assert bool((td >= 10.0).any()) and bool(ctx['valid'].any())
        hm = ctx['ray_mask']
        assert bool((hm[1:] != hm[:-1]).sum() > 100)      # misses interleaved with hits
    elif name == 'no_sign':
        sdf = c['ref']['sdf']
        change = ((sdf[:, 1:] * sdf[:, :-1]) < 0).any(1)
        assert int(change.sum()) > 10 and int((~change).sum()) > 10


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('name', CASES)
def test_step_vs_float64(refs, name, mode):
    rep, c, _, q_err = run_case(refs, name, mode)
    _case_property(name, c)
    _check(rep, c, q_err, mode, name)


@pytest.mark.parametrize('mode', MODES)
def test_pose_only_vs_float64(refs, mode):
    """Tracking pass (freeze_map_grads: d_embeddings and d_decoder NULL): the rays alone."""
    rep, c, g, q_err = run_case(refs, 'bench', mode, need_map=False)
    assert g['d_emb'] is None and all(t is None for t in g['d_dec'])
    assert 'entry' not in rep and 'd_w0' not in rep and 'd_rays_d' in rep
    _check(rep, c, q_err, mode, 'pose-only')


@pytest.mark.parametrize('mode', MODES)
def test_map_only_vs_float64(refs, mode):
    rep, c, g, q_err = run_case(refs, 'bench', mode, need_rays=False)
    assert g['d_rays_o'] is None and g['d_rays_d'] is None
    assert 'entry' in rep and 'd_wc0' in rep and 'd_rays_o' not in rep
    _check(rep, c, q_err, mode, 'map-only')
