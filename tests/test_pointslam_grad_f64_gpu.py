"""Point-SLAM render-and-optimise step (xrd_pointslam_step through ConvOnet2._launch, all four
GEMM arithmetic modes) against the float64 replay of oracle/pointslam_f64.py: every row of
d_geo_feats and d_col_feats (rows no sample touches exactly 0), every element of the 25
colour-decoder gradients (B_rel included), every ray and component, both loss terms, rgb, depth
and uncertainty; z, the neighbour ids and counts and valid_ray_mask bit for bit.  The
whole-tensor relative L2 of test_pointslam_gpu.py lets a wrong weight on one neighbour slot, a
lost atomic on one point or one wrong ray through; these checks do not.

Gates (per GEMM mode): about 4x the worst ratio over all cases below (test_report_worst prints
that column), compared with the ratio the mutations of test_pointslam_f64_reference_cpu.py
produce at that check:

  mode  check   worst on the H100 (case)   gate     mutation floor (CPU)
  0     feat    2.2e-9  (bench)            1e-8     1.3e-5  one slot's weight from slot j + 1
        weight  1.0e-4  (one)              4e-4     6.0e-4  most exposed element x (1 + 1e-3)
        ray     4.0e-11 (trk_even)         2e-10    1.1e-7  d_rays_d without z, one ray
        loss    5.1e-6  (trk_even)         2e-5
        fwd     6.9e-6  (depth_edges)      3e-5
  1, 3  feat    2.9e-9  (bench)            1.2e-8   as above
        weight  3.6e-4  (p_mixed)          1.5e-3   5.6e-3  -1 slots weighted
        ray     1.7e-10 (trk_even)         7e-10    as above
        loss    5.1e-6  (trk_even)         2e-5
        fwd     6.6e-6  (depth_edges)      3e-5
  2     feat    1.1e-6  (depth_edges)      4.5e-6
        weight  0.24    (p_mixed)          1.0
        ray     8.8e-8  (trk_even)         3.5e-7
        loss    7.6e-4  (shared)           3e-3
        fwd     1.8e-3  (trk_bench)        7.5e-3
  Other floors: colour features masked 0.11 (weight), radius test `>=` 7.9e-2 (weight),
  uncertainty not detached 5e-4 (feat), composite suffix term dropped 1.6e-4 (feat), weights
  normalised without the sum term 1.9e-6 (ray), neighbour ray copied 5.4e-7 (ray); frustum mask
  ignored for geometry features, depth gradient on zero-depth rays and the upper median land
  where nothing may (inf).
  Not seen (NOT_SEEN in the CPU file): three stale pad columns in the neighbour weight gradients
  (2.5e-7) and the last 64 columns of a weight reduction dropped (3.9e-5) stay under every weight
  gate: the weight gates are set by batches of a few hundred samples (one, p_mixed), where an
  element is a sum of few terms that carry the fp32 error of sin(2 pi p B) at ~300 rad through
  softplus(beta = 100); batches of 1500 samples and more stay near 1e-5.  Occupancy gradient on
  samples without neighbours moves a ray by 8.7e-12 (their alpha is sigmoid(-10)).  A 1e-3
  change of one element is seen by mode 0 only, and only on the most exposed elements (smallest
  over the 25 tensors: 2e-10).  The per-element weight check therefore resolves structural
  faults (a masked or shifted input, a wrong radius test, a weighted -1 slot), not single lost
  columns.  Plain TF32 (mode 2) sees only the faults above its gates; its weight gate is vacuous.
  Mode 1 equals mode 3 below 512 columns (both run k_gemm_tc<true>); at the bench shape mode 1 is
  the wgmma kernel throughout, its 144 = 128 + 16 row split included.
  Rays whose loss decisions differ from float64: 0 in modes 0, 1, 3 (cap 0); mode 2 a few of
  5000 (cap 6); trk_clamp 12 to 13 of 600 in every mode (depth == target to the last bit).
  Exempt share (ambiguous ReLU): rows 3.0 % and rays 2.8 % at the bench shape; at B std 25 (b25,
  geometry embedding x 20) rows 3.1 %, rays 3.2 %.  Rows an ambiguous sample touches are still
  judged, beyond twice that sample's share of the row's bound (shared: all 12 rows).
  The sample points p = o + d * z of the step itself are not an output: z and valid_ray_mask are
  compared bit for bit, the kNN through the explicit-query entry point on the replay's fp32 p,
  and p_tail, mask and trk_bench start every ray at its own non-zero origin, so that a different
  rounding of p inside the step would move neighbour sets and show in the gradients.
  Measured on one H100 80GB HBM3 at a 700 W power limit; the file runs in about 16 s there.

The fp32 CPU oracle itself stays within feat 2.7e-9, weight 3.1e-5, ray 4.1e-11, loss 9.4e-7 and
forward 4.4e-7 of float64 (test_pointslam_f64_reference_cpu.py).
"""
import contextlib

import pytest
import torch

pytestmark = pytest.mark.gpu

# ReLU ambiguity threshold |pre| / sum|terms| of the geometry decoder.  It runs in fp32 SIMT
# under every GEMM mode (the mode selects the arithmetic of the colour stage's GEMMs only).
AMB = {0: 1e-5, 1: 1e-5, 2: 1e-5, 3: 1e-5}
GATES = {
    0: dict(feat=1e-8, weight=4e-4, ray=2e-10, loss=2e-5, fwd=3e-5),
    1: dict(feat=1.2e-8, weight=1.5e-3, ray=7e-10, loss=2e-5, fwd=3e-5),
    2: dict(feat=4.5e-6, weight=1.0, ray=3.5e-7, loss=3e-3, fwd=7.5e-3),
    3: dict(feat=1.2e-8, weight=1.5e-3, ray=7e-10, loss=2e-5, fwd=3e-5),
}
MODES = (0, 1, 2, 3)
STRICT_MODES = (0, 1, 3)
# rays whose loss decisions may differ between the kernel and float64, per mode; trk_clamp has
# its own cap (FLIP_CAP_CASE in the CPU file)
MAX_FLIP_RAYS = {0: 0, 1: 0, 2: 6, 3: 0}
# trk_median: the one ray in the loss renders its target depth to 2e-6, so |D - d| (the loss value)
# and the few-term colour sums carry the fp32 rounding of depth itself.  The case is there for the
# mask: ray 0 lies outside it and every entry only ray 0 reaches must be exactly 0
CASE_GATES = {'trk_median': dict(weight=1.0, loss=1.0)}
# cases large enough for the share of ambiguous-ReLU exemptions to be asserted small
COVERAGE_CASES = ('bench', 'trk_bench', 'mask', 'p_tail')
SEEN = {}              # (case, mode) -> worst ratios; test_report_worst prints the table's column


@contextlib.contextmanager
def gemm_mode(mode):
    from xrdslam_b200 import _cabi
    lib = _cabi.lib()
    _cabi.check('xrd_debug_gemm_mode', lib.xrd_debug_gemm_mode(mode))
    try:
        yield
    finally:
        lib.xrd_debug_gemm_mode(1)


class _Refs:
    """Per case: the CUDA model, the device batch and the float64 replay, each built once."""

    def __init__(self, dev):
        self.dev, self.cache = dev, {}

    def get(self, name):
        if name in self.cache:
            return self.cache[name]
        from helpers import pointslam_from_golden
        from oracle import pointslam_f64 as F
        from test_pointslam_f64_reference_cpu import CASES, golden_dict
        dev = self.dev
        b = CASES[name]()
        g = golden_dict(b)
        cfg = dict(F.DEFAULT_CFG, **b['cfg'])
        model = pointslam_from_golden(g, 'b200', dev)
        mc = model.config
        mc.rendering_n_surface = cfg['S']
        mc.rendering_sigmoid_coef_mapper = cfg['coef']
        mc.tracking_handle_dynamic = cfg['handle_dynamic']
        mc.tracking_use_color_in_tracking = cfg['use_color_trk']
        mc.mapping_w_color_loss = mc.tracking_w_color_loss = cfg['w_color']
        model._t_surface = torch.linspace(0.0, 1.0, steps=cfg['S'], device=dev)
        npc = model.neural_point_cloud
        if b['fmask'] is not None:
            npc.set_mask(b['fmask'])
        d = {k: b[k].to(dev) for k in ('rays_o', 'rays_d', 'target_d', 'target_s', 'radius')}
        rf = torch.from_numpy(g['rand_feat']).to(dev)
        rfc = torch.from_numpy(g['rand_feat_color']).to(dev)
        ctx = F.prepare(d['rays_o'], d['rays_d'], d['target_d'], d['target_s'], d['radius'],
                        b['cloud'], b['fmask'], b['cfg'], far=F.far_end(d['target_d']), device=dev)
        # the kernel's own kNN on the replay's fp32 sample points: ids, distances and counts
        Dk, Ik, nk = npc.find_neighbors(ctx['p32'], d['radius'].repeat_interleave(cfg['S']))
        assert torch.equal(Ik.long(), ctx['I']) and torch.equal(nk.long(), ctx['nn'])
        assert torch.equal(Dk[Ik >= 0], ctx['D32'][ctx['I'] >= 0])
        ref = F.replay_step(ctx, F.params_from_model(model, rf, rfc))
        self.cache[name] = dict(model=model, d=d, rf=rf, rfc=rfc, ctx=ctx, ref=ref, cfg=cfg)
        return self.cache[name]


@pytest.fixture(scope='module')
def refs(cuda_dev):
    return _Refs(cuda_dev)


def launch(c, need_rays=True, need_feats=True, need_cdec=True):
    model, d, cfg = c['model'], c['d'], c['cfg']
    color = cfg['stage'] == 'color'
    model._z_capture = torch.empty(c['ctx']['P'], device=d['rays_o'].device)
    out, g = model._launch(cfg['stage'], cfg['is_mapping'], d['rays_o'], d['rays_d'],
                           d['target_s'], d['target_d'], d['radius'], c['rf'], True,
                           need_rays=need_rays, need_feats=need_feats, rand_feat_color=c['rfc'],
                           need_col_feats=color and need_feats, need_cdec=color and need_cdec)
    torch.cuda.synchronize()
    out['z'] = model._z_capture.view(-1, cfg['S'])
    model._z_capture = None
    return out, g


def run_case(refs, name, mode, **need):
    """One step under GEMM mode ``mode`` -> (compare report, case, outputs, gradients)."""
    from oracle import pointslam_f64 as F
    c = refs.get(name)
    ctx = c['ctx']
    with gemm_mode(mode):
        out, g = launch(c, **need)
    assert torch.equal(out['z'], ctx['z32'])
    assert torch.equal(out['valid_ray_mask'], ctx['valid'])
    for k, v in g.items():
        for t in (v if isinstance(v, list) else [v]):
            assert t is None or bool(torch.isfinite(t).all()), k
    cand = dict(g, losses=out['losses'], rgb=out['rgb'], depth=out['depth'],
                uncertainty=out['uncertainty'])
    rep, ref = F.compare(c['ref'], cand, AMB[mode])
    SEEN[(name, mode) + tuple(sorted(need))] = dict(F.worst(rep), flip=rep['n_flip_rays'],
                                                   near=rep['n_near'], rows=rep.get('exempt_rows'),
                                                   rays=rep['exempt_rays'])
    return rep, c, out, g, ref


def _check(rep, mode, name):
    from oracle import pointslam_f64 as F
    from test_pointslam_f64_reference_cpu import FLIP_CAP_CASE
    cap = FLIP_CAP_CASE.get(name, MAX_FLIP_RAYS[mode])
    assert rep['n_flip_rays'] <= cap and rep['n_near'] == 0, rep
    if name.split('/')[0] in COVERAGE_CASES:   # elsewhere the share is reported, not coverage
        assert rep.get('exempt_rows', 0.0) < 0.05 and rep['exempt_rays'] < 0.05, rep
    bad = F.failures(rep, dict(GATES[mode], **CASE_GATES.get(name, {})))
    assert not bad, (name, mode, bad)


CASE_NAMES = ('bench', 'p_small', 'p_mixed', 'p_tail', 'one', 'S2', 'S3', 'S8', 'S16', 'mask',
              'sparse', 'on_point', 'on_radius', 'shared', 'depth_edges', 'depth_zero', 'trk_even',
              'trk_nodyn', 'trk_clamp', 'trk_median', 'trk_nocolor', 'trk_bench', 'trk_geo', 'b25')


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('name', CASE_NAMES)
def test_step_vs_float64(refs, name, mode):
    from test_pointslam_f64_reference_cpu import case_property
    rep, c, out, g, ref = run_case(refs, name, mode)
    case_property(name, c['ctx'], ref)
    _check(rep, mode, name)
    if name == 'depth_zero':   # no ray carries a loss: every gradient is exactly 0
        assert float(out['losses'].abs().sum()) == 0.0
        assert all(float(t.abs().sum()) == 0.0 for t in
                   [g['d_geo_feats'], g['d_col_feats'], g['d_rays_o'], g['d_rays_d']] + g['d_cdec'])
    if name == 'b25':
        print(f"\n  b25 mode {mode}: exempt rows {rep['exempt_rows']:.3f}, "
              f"rays {rep['exempt_rays']:.3f}")


def test_case_list_is_complete():
    from test_pointslam_f64_reference_cpu import CASES
    assert sorted(CASE_NAMES) == sorted(CASES)


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('subset', ['rays', 'feats', 'no_cdec'])
def test_gradient_subsets(refs, mode, subset):
    """NULL members of XrdPointGrads: rays only (tracking), features only, no colour-decoder
    gradients.  What is still computed passes the gates; outputs, losses and the ray gradients
    (no atomics on their path) equal the full run's bit for bit."""
    need = dict(rays=dict(need_feats=False, need_cdec=False), feats=dict(need_rays=False,
                need_cdec=False), no_cdec=dict(need_cdec=False))[subset]
    _, _, out0, g0, _ = run_case(refs, 'mask', mode)
    rep, c, out, g, _ = run_case(refs, 'mask', mode, **need)
    _check(rep, mode, 'mask/' + subset)
    assert g['d_cdec'] is None
    assert (g['d_rays_o'] is None) == (subset == 'feats')
    assert (g['d_geo_feats'] is None) == (g['d_col_feats'] is None) == (subset == 'rays')
    for k in ('rgb', 'depth', 'uncertainty', 'losses', 'valid_ray_mask'):
        assert torch.equal(out[k], out0[k]), k
    if subset != 'feats':
        assert torch.equal(g['d_rays_o'], g0['d_rays_o'])
        assert torch.equal(g['d_rays_d'], g0['d_rays_d'])


def test_tracking_ray_limit(refs):
    """Tracking takes 8192 rays (the single-block median of k_loss; trk_geo runs them) and
    refuses 8193 with XRD_E_SHAPE."""
    c = refs.get('trk_geo')
    assert c['ctx']['R'] == 8192
    d = {k: torch.cat([v, v[:1]]) for k, v in c['d'].items()}
    with pytest.raises(RuntimeError, match='XRD_E_SHAPE|shape'):
        c['model']._launch('geometry', False, d['rays_o'], d['rays_d'], d['target_s'],
                           d['target_d'], d['radius'], c['rf'], True, need_rays=True)


def test_report_worst(capsys):
    """Prints the worst ratio per mode and check over the cases run before it, with its case (the
    'worst on the H100' column of the table above)."""
    with capsys.disabled():
        for mode in MODES:
            for kind in ('feat', 'weight', 'ray', 'loss', 'fwd'):
                rows = [(v[kind], k[0]) for k, v in SEEN.items()
                        if k[1] == mode and kind not in CASE_GATES.get(k[0], {})]
                if rows:
                    print(f'  worst mode {mode} {kind:6s} %.2g (%s)' % max(rows))
