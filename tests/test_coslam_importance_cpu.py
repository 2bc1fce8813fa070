"""Co-SLAM importance sampling (training_n_importance > 0): the importance oracle against the
reference's own JointEncoding with training_n_importance > 0 (live, and through the committed
fixture tests/golden/coslam_importance_step.npz), with the deterministic (training_perturb = 0)
and the random draw of sample_pdf; the model's configuration checks and C structs.  No GPU
needed."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from helpers import BOUND, coslam_pair, make_rays

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden',
                      'coslam_importance_step.npz')
R_CASE = 16
OUT_KEYS = ('rgb', 'depth', 'disp_map', 'acc_map', 'depth_var', 'z_vals', 'raw')
IMP_KEYS = ('rgb0', 'disp0', 'acc0', 'depth0', 'depth_var0', 'z_std')
LOSS_KEYS = ('rgb_loss', 'depth_loss', 'sdf_loss', 'fs_loss')
WEIGHTS = (('sdf0', 'decoder.sdf_net.model.0.weight'), ('sdf1', 'decoder.sdf_net.model.2.weight'),
           ('col0', 'decoder.color_net.model.0.weight'), ('col1', 'decoder.color_net.model.2.weight'))
# (N, det) of the fixture; the live comparison runs all four
GOLDEN_CASES = ((5, True), (16, False))
CASES = ((5, False), (5, True), (16, False), (16, True))


def importance_case(N, det):
    """One-grid oracle with helpers.coslam_pair's seeded parameters, R_CASE rays, and the draws
    the reference makes after torch.manual_seed(9): the coarse jitter torch.rand(R, 43) (none
    when det: training_perturb = 0) and sample_pdf's torch.rand(R, N) (its linspace when det)."""
    from oracle.coslam_importance import det_u
    ora, _ = coslam_pair('cpu')
    ora.cfg.perturb = 0 if det else 1
    rays_o, rays_d, ts, td, _ = make_rays(R_CASE, seed=5)
    torch.manual_seed(9)
    if det:
        noise, u = torch.zeros(R_CASE, 43), det_u(N).expand(R_CASE, N)
    else:
        noise = torch.rand(R_CASE, 43)
        u = torch.rand(R_CASE, N)
    return ora, (rays_o, rays_d, ts, td, noise, u)


def _record(out, ld, table, weights, rays):
    np_ = lambda t: t.detach().cpu().numpy()
    rec = {k: np_(out[k]) for k in OUT_KEYS + IMP_KEYS}
    rec['losses'] = np.array([float(ld[k].detach()) for k in LOSS_KEYS], dtype=np.float64)
    gr = table.grad.detach().reshape(-1, 2)
    idx = torch.nonzero(gr.abs().sum(-1)).reshape(-1)
    rec['d_table.idx'] = idx.numpy().astype(np.int32)
    rec['d_table.val'] = np_(gr[idx])
    for name, t in weights.items():
        rec[name] = np_(t.grad)
    rec['d_rays_o'], rec['d_rays_d'] = np_(rays[0].grad), np_(rays[1].grad)
    return rec


def run_oracle_step(N, det):
    from oracle import coslam_importance as CI
    ora, (rays_o, rays_d, ts, td, noise, u) = importance_case(N, det)
    rays_o.requires_grad_(True)
    rays_d.requires_grad_(True)
    out, ld, tot = CI.step(ora, rays_o, rays_d, ts, td, noise, u)
    tot.backward()
    return _record(out, ld, ora.embed_fn.params, {'d_' + n: getattr(ora, n).weight
                                                   for n, _ in WEIGHTS}, (rays_o, rays_d))


def run_reference_step(N, det):
    """The reference's JointEncoding(training_n_importance=N) on importance_case()'s parameters
    and rays (needs the reference checkout)."""
    from oracle import ref_harness
    ora, (rays_o, rays_d, ts, td, noise, u) = importance_case(N, det)
    ref = ref_harness.ref_joint_encoding(torch.from_numpy(BOUND), training_n_importance=N,
                                         training_perturb=0 if det else 1)
    sd = ref.state_dict()
    with torch.no_grad():
        ref.embed_fn.params.copy_(ora.embed_fn.params)
        for name, key in WEIGHTS:
            sd[key].copy_(getattr(ora, name).weight)
    rays_o.requires_grad_(True)
    rays_d.requires_grad_(True)
    torch.manual_seed(9)  # the reference draws what importance_case drew
    inp = dict(rays_o=rays_o, rays_d=rays_d, target_s=ts, target_d=td, first=True)
    out = ref(inp)
    assert set(IMP_KEYS) <= set(out)
    ld = ref.get_loss_dict(out, inp, False, 0)
    assert set(ld) == set(LOSS_KEYS)
    sum(ld.values()).backward()
    params = dict(ref.named_parameters())
    rec = _record(out, ld, ref.embed_fn.params, {'d_' + n: params[k] for n, k in WEIGHTS},
                  (rays_o, rays_d))
    rec.update(rays_o=rays_o.detach().numpy(), rays_d=rays_d.detach().numpy(),
               target_s=ts.numpy(), target_d=td.numpy(), noise=noise.numpy(), u=u.numpy())
    return rec


def _compare(got, want):
    for k in OUT_KEYS + IMP_KEYS:
        assert np.array_equal(got[k], want[k]), k
    assert np.allclose(got['losses'], want['losses'], rtol=1e-6, atol=0)
    assert np.array_equal(got['d_table.idx'], want['d_table.idx'])
    assert np.allclose(got['d_table.val'], want['d_table.val'], rtol=1e-5, atol=1e-9)
    for k in ['d_' + n for n, _ in WEIGHTS] + ['d_rays_o', 'd_rays_d']:
        assert np.allclose(got[k], want[k], rtol=1e-5, atol=1e-9), k


@pytest.mark.needs_reference
@pytest.mark.parametrize('N,det', CASES)
def test_oracle_matches_reference_class_live(N, det):
    """The importance oracle == the reference's JointEncoding(training_n_importance=N): outputs,
    the coarse outputs, z_std, the four loss terms and every gradient bit-identical (the two run
    the same reductions in this process)."""
    ref, ora = run_reference_step(N, det), run_oracle_step(N, det)
    _compare(ora, ref)
    for k in ('d_table.val', 'd_sdf0', 'd_sdf1', 'd_col0', 'd_col1', 'd_rays_o', 'd_rays_d',
              'losses'):
        assert np.array_equal(ora[k], ref[k]), k
    assert ora['z_vals'].shape == (R_CASE, 43 + N)


@pytest.mark.parametrize('N,det', GOLDEN_CASES)
def test_oracle_matches_golden_reference_step(N, det):
    """The importance oracle reproduces the committed reference fixture."""
    g = np.load(GOLDEN)
    pre = f'n{N}_det{int(det)}/'
    g = {k[len(pre):]: g[k] for k in g.files if k.startswith(pre)}
    assert g
    _, (rays_o, rays_d, ts, td, noise, u) = importance_case(N, det)
    for k, v in (('rays_o', rays_o), ('rays_d', rays_d), ('target_s', ts), ('target_d', td),
                 ('noise', noise), ('u', u)):
        assert np.array_equal(g[k], v.numpy()), k
    got = run_oracle_step(N, det)
    _compare(got, g)
    # the fine pass marches more samples than the coarse one, and its sdf / fs terms count
    # over them
    assert got['z_vals'].shape == (R_CASE, 43 + N)
    assert np.all(np.diff(got['z_vals'], axis=-1) >= 0)


def test_sample_pdf_det_samples_sorted_and_inside_bins():
    """sample_pdf on the coarse weights: samples lie between the first and last bin midpoint,
    and the det draw gives sorted samples."""
    from oracle import coslam_importance as CI
    ora, (rays_o, rays_d, ts, td, noise, u) = importance_case(16, True)
    with torch.no_grad():
        out = CI.render_rays(ora, rays_o, rays_d, td, noise, u)
    zc = out['coarse']['z_vals']
    mid = .5 * (zc[..., 1:] + zc[..., :-1])
    zs = out['z_samples']
    assert torch.all(zs >= mid[:, :1]) and torch.all(zs <= mid[:, -1:])
    assert torch.all(zs[:, 1:] >= zs[:, :-1])


def _model(**cfg):
    from xrdslam_b200.camera import Camera
    from xrdslam_b200.joint_encoding import JointEncodingConfig
    return JointEncodingConfig(**cfg).setup(
        camera=Camera(320., 320., 319.5, 239.5, 640, 480), bounding_box=BOUND)


def test_config_accepts_importance_sampling():
    from oracle.coslam_importance import det_u
    from xrdslam_b200.joint_encoding import IMPORTANCE_KEYS, OUT_KEYS as MODEL_OUT_KEYS
    m = _model(training_n_importance=16)
    assert torch.equal(m._lin_u, det_u(16))
    assert m._out_keys() == MODEL_OUT_KEYS + IMPORTANCE_KEYS
    assert set(IMPORTANCE_KEYS) == set(IMP_KEYS)
    assert _model()._out_keys() == MODEL_OUT_KEYS and _model()._lin_u is None
    # the largest N that fits: 43 + 213 = 256 samples per ray (224 with a colour grid)
    _model(training_n_importance=213)
    _model(training_n_importance=181, oneGrid=False)


@pytest.mark.parametrize('cfg,limit', [(dict(training_n_importance=214), 256),
                                       (dict(training_n_importance=182, oneGrid=False), 224)])
def test_config_rejects_importance_that_does_not_fit(cfg, limit):
    with pytest.raises(ValueError, match=f'march .* = {43 + cfg["training_n_importance"]} '
                                         f'samples per ray; the fused kernels take at most {limit}'):
        _model(**cfg)
    with pytest.raises(ValueError, match='>= 0'):
        _model(training_n_importance=-1)
    with pytest.raises(NotImplementedError, match='tcnn_network'):
        _model(tcnn_network=True)


def test_importance_c_structs():
    """n_importance is the last field of XrdCoslamCfg (earlier fields keep their offsets), and
    the importance step's struct carries what the model puts in it."""
    from xrdslam_b200 import _cabi
    cfg = _cabi.XrdCoslamCfg
    assert cfg.n_importance.offset == cfg.seed_dev.offset + C.sizeof(C.c_void_p)
    assert cfg.seed_dev.offset == 112 and C.sizeof(cfg) == 128  # as the C compiler lays it out
    q = _cabi.XrdCoslamImportance
    assert [n for n, _ in q._fields_] == [
        'n_rays', 'n_samples', 'n_importance', 'det', 'trunc', 'depth_trunc', 'z_vals', 'raw',
        'target_d', 'u', 'lin_u', 'seed', 'seed_dev', 'z_fine', 'z_samples', 'z_std',
        'counts_out']
    assert q.z_vals.offset == 24 and q.counts_out.offset == 104 and C.sizeof(q) == 112
    m = _model(training_n_importance=16, training_perturb=0)
    z, raw = torch.zeros(4, 43), torch.zeros(4, 43, 4)
    b, s = m._importance_struct(4, 43, 'cpu', z, raw, seed=7)
    assert (s.n_rays, s.n_samples, s.n_importance, s.det, s.seed) == (4, 43, 16, 1, 7)
    assert b['z_vals'].shape == (4, 59) and b['z_samples'].shape == (4, 16)
    assert s.lin_u == m._lin_u.data_ptr() and s.z_fine == b['z_vals'].data_ptr()
    assert not s.u and not s.counts_out and not s.seed_dev
    assert m._cfg_struct(59, phase=2, n_importance=16).n_importance == 16
