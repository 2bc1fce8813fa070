"""Co-SLAM with a separate colour hash grid (oneGrid=False): the two-grid oracle against the
reference's own JointEncoding(oneGrid=False) (live, and through the committed fixture
tests/golden/coslam_color_grid_step.npz), and the model's parameters, groups and colour-grid
layout against the oracle.  No GPU needed."""
import os

import numpy as np
import pytest
import torch

from helpers import BOUND, make_rays

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden',
                      'coslam_color_grid_step.npz')
R_CASE = 16
OUT_KEYS = ('rgb', 'depth', 'disp_map', 'acc_map', 'depth_var', 'z_vals', 'raw')
LOSS_KEYS = ('rgb_loss', 'depth_loss', 'sdf_loss', 'fs_loss')
# (oracle attribute, reference / CUDA-model state-dict name) of the four decoder weights
WEIGHTS = (('sdf0', 'decoder.sdf_net.model.0.weight'), ('sdf1', 'decoder.sdf_net.model.2.weight'),
           ('col0', 'decoder.color_net.model.0.weight'), ('col1', 'decoder.color_net.model.2.weight'))


def color_grid_case():
    """Two-grid oracle with seeded parameters (tables U(-0.3, 0.3), weights N(0, 1/fan_in)) and
    the inputs of the comparison with the reference: R_CASE rays and the perturbation noise the
    reference draws after torch.manual_seed(9)."""
    from oracle.coslam_color_grid import CoslamColorGridOracle
    ora = CoslamColorGridOracle(BOUND)
    with torch.no_grad():
        for seed, enc in ((21, ora.embed_fn), (22, ora.embed_fn_color)):
            g = torch.Generator().manual_seed(seed)
            enc.params.copy_((torch.rand(enc.params.shape, generator=g) * 2 - 1) * 0.3)
        g = torch.Generator().manual_seed(23)
        for name, _ in WEIGHTS:
            lin = getattr(ora, name)
            lin.weight.copy_(torch.randn(lin.weight.shape, generator=g) / np.sqrt(lin.weight.shape[1]))
    rays_o, rays_d, ts, td, _ = make_rays(R_CASE, seed=5)
    torch.manual_seed(9)
    noise = torch.rand(R_CASE, 43)
    return ora, (rays_o, rays_d, ts, td, noise)


def _record(out, ld, tables, weights, rays):
    """{key: array} of one step: outputs, losses, sparse table gradients, dense weight and ray
    gradients."""
    np_ = lambda t: t.detach().cpu().numpy()
    rec = {k: np_(out[k]) for k in OUT_KEYS}
    rec['losses'] = np.array([float(ld[k].detach()) for k in LOSS_KEYS], dtype=np.float64)
    for name, t in tables.items():
        gr = t.grad.detach().reshape(-1, 2)
        idx = torch.nonzero(gr.abs().sum(-1)).reshape(-1)
        rec[name + '.idx'] = idx.numpy().astype(np.int32)
        rec[name + '.val'] = np_(gr[idx])
    for name, t in weights.items():
        rec[name] = np_(t.grad)
    rec['d_rays_o'], rec['d_rays_d'] = np_(rays[0].grad), np_(rays[1].grad)
    return rec


def run_oracle_step():
    ora, (rays_o, rays_d, ts, td, noise) = color_grid_case()
    rays_o.requires_grad_(True)
    rays_d.requires_grad_(True)
    out, ld, tot = ora.step(rays_o, rays_d, ts, td, noise, False, True)
    tot.backward()
    return _record(out, ld, {'d_table': ora.embed_fn.params, 'd_table_color': ora.embed_fn_color.params},
                   {'d_' + n: getattr(ora, n).weight for n, _ in WEIGHTS}, (rays_o, rays_d))


def run_reference_step():
    """The reference's JointEncoding(oneGrid=False) on color_grid_case()'s parameters and rays
    (needs the reference checkout)."""
    from oracle import ref_harness
    ora, (rays_o, rays_d, ts, td, noise) = color_grid_case()
    ref = ref_harness.ref_joint_encoding(torch.from_numpy(BOUND), oneGrid=False)
    sd = ref.state_dict()
    with torch.no_grad():
        ref.embed_fn.params.copy_(ora.embed_fn.params)
        ref.embed_fn_color.params.copy_(ora.embed_fn_color.params)
        for name, key in WEIGHTS:
            sd[key].copy_(getattr(ora, name).weight)
    rays_o.requires_grad_(True)
    rays_d.requires_grad_(True)
    torch.manual_seed(9)  # the reference draws the same noise as color_grid_case
    inp = dict(rays_o=rays_o, rays_d=rays_d, target_s=ts, target_d=td, first=True)
    out = ref(inp)
    ld = ref.get_loss_dict(out, inp, False, 0)
    assert set(ld) == set(LOSS_KEYS)
    sum(ld.values()).backward()
    params = dict(ref.named_parameters())
    rec = _record(out, ld, {'d_table': ref.embed_fn.params, 'd_table_color': ref.embed_fn_color.params},
                  {'d_' + n: params[k] for n, k in WEIGHTS}, (rays_o, rays_d))
    rec.update(rays_o=rays_o.detach().numpy(), rays_d=rays_d.detach().numpy(),
               target_s=ts.numpy(), target_d=td.numpy(), noise=noise.numpy())
    return rec


def _compare(got, want, exact):
    for k in OUT_KEYS:
        if exact:
            assert np.array_equal(got[k], want[k]), k
        else:
            assert np.allclose(got[k], want[k], rtol=0, atol=1e-6), k
    # losses and gradients are reductions whose order can follow the host's SIMD width
    assert np.allclose(got['losses'], want['losses'], rtol=1e-6, atol=0)
    for k in ('d_table', 'd_table_color'):
        assert np.array_equal(got[k + '.idx'], want[k + '.idx']), k
        assert np.allclose(got[k + '.val'], want[k + '.val'], rtol=1e-5, atol=1e-9), k
    for k in ['d_' + n for n, _ in WEIGHTS] + ['d_rays_o', 'd_rays_d']:
        assert np.allclose(got[k], want[k], rtol=1e-5, atol=1e-9), k


@pytest.mark.needs_reference
def test_oracle_matches_reference_class_live():
    """The two-grid oracle == the reference's JointEncoding(oneGrid=False): outputs bit-identical,
    losses and every gradient (both tables per entry, the four weights, the rays) equal up to the
    order of reductions."""
    ref, ora = run_reference_step(), run_oracle_step()
    _compare(ora, ref, exact=True)
    # in this process the two run the same reductions: bit-identical throughout
    for k in ('d_table.val', 'd_table_color.val', 'd_sdf0', 'd_sdf1', 'd_col0', 'd_col1',
              'd_rays_o', 'd_rays_d'):
        assert np.array_equal(ora[k], ref[k]), k
    assert np.array_equal(ora['losses'], ref['losses'])


def test_oracle_matches_golden_reference_step():
    """The two-grid oracle reproduces the committed reference fixture."""
    g = np.load(GOLDEN)
    g = {k: g[k] for k in g.files}
    ora, (rays_o, rays_d, ts, td, noise) = color_grid_case()
    for k, v in (('rays_o', rays_o), ('rays_d', rays_d), ('target_s', ts), ('target_d', td),
                 ('noise', noise)):
        assert np.array_equal(g[k], v.numpy()), k
    assert g['d_table_color.idx'].size > 0 and np.abs(g['d_table_color.val']).max() > 0
    _compare(run_oracle_step(), g, exact=True)


def _model(**cfg):
    from xrdslam_b200.camera import Camera
    from xrdslam_b200.joint_encoding import JointEncodingConfig
    return JointEncodingConfig(**{'oneGrid': False, **cfg}).setup(
        camera=Camera(320., 320., 319.5, 239.5, 640, 480), bounding_box=BOUND)


def test_color_grid_layout_matches_oracle():
    from oracle.coslam_color_grid import CoslamColorGridOracle
    from oracle.tcnn_restated import hashgrid_level_table
    model, ora = _model(), CoslamColorGridOracle(BOUND)
    assert model.resolution_color == ora.resolution_color == 81
    t = ora.embed_fn_color.table
    g = model.embed_fn_color.layout
    assert int(g.n_entries) == 653_976 and 2 * int(g.n_entries) == t['n_params']
    assert model.embed_fn_color.params.numel() == 1_307_952
    assert all(float(np.float32(g.scale[l])) == float(t['scale'][l]) for l in range(16))
    for k in ('resolution', 'size', 'offset', 'hashed'):
        assert [int(getattr(g, k)[l]) for l in range(16)] == [int(v) for v in t[k]], k
    # levels 0-8 dense, 9-15 hashed
    assert [int(g.hashed[l]) for l in range(16)] == [0] * 9 + [1] * 7
    assert float(model.embed_fn_color.params.detach().abs().max()) <= 1e-4
    # voxel_color > 10 is the resolution itself
    assert _model(voxel_color=40).resolution_color == 40
    ref = hashgrid_level_table(16, 2, 16, 16, np.exp2(np.log2(40 / 16) / 15))
    assert 2 * int(_model(voxel_color=40).embed_fn_color.layout.n_entries) == ref['n_params']


def test_color_grid_parameters_and_groups():
    model = _model()
    sd = model.state_dict()
    assert tuple(sd['decoder.color_net.model.0.weight'].shape) == (32, 95)
    assert tuple(sd['decoder.color_net.model.2.weight'].shape) == (3, 32)
    assert tuple(sd['decoder.sdf_net.model.0.weight'].shape) == (32, 80)
    assert tuple(sd['embed_fn_color.params'].shape) == (1_307_952,)
    groups = model.get_param_groups()
    assert set(groups) == {'decoder', 'embed_fn', 'embed_fn_color'}
    assert groups['embed_fn_color'][0] is model.embed_fn_color.params
    one = _model(oneGrid=True)
    assert set(one.get_param_groups()) == {'decoder', 'embed_fn'}
    assert tuple(one.state_dict()['decoder.color_net.model.0.weight'].shape) == (32, 63)


def test_color_grid_c_structs():
    """The colour grid travels in XrdCoslamMlp.grid_color; NULL keeps the one-grid path."""
    import ctypes as C
    model = _model()
    mlp = model._mlp_struct(model._weights())
    assert bool(mlp.grid_color)
    assert mlp.grid_color.contents.n_entries == model.embed_fn_color.layout.n_entries
    assert mlp.grid_color.contents.table == model.embed_fn_color.params.data_ptr()
    assert mlp.grid_color.contents.bbox_max[1] == BOUND[1, 1]
    one = _model(oneGrid=True)
    assert not bool(one._mlp_struct(one._weights()).grid_color)
    from xrdslam_b200._cabi import XrdCoslamGrads
    assert XrdCoslamGrads.d_table_color.offset == C.sizeof(XrdCoslamGrads) - C.sizeof(C.c_void_p)


def test_oracle_color_branch_uses_color_grid():
    """Only the colour output depends on the colour table."""
    from oracle.coslam_color_grid import CoslamColorGridOracle
    ora = CoslamColorGridOracle(BOUND)
    x = torch.rand(64, 3, generator=torch.Generator().manual_seed(0))
    a = ora.query_color_sdf(x).detach()
    with torch.no_grad():
        ora.embed_fn_color.params.mul_(50.0)
    b = ora.query_color_sdf(x).detach()
    assert torch.equal(a[:, 3], b[:, 3])
    assert not torch.equal(a[:, :3], b[:, :3])
