"""Parity of the NICE-SLAM CUDA path (C-ABI) against oracle/nice.py (itself pinned to the
reference's ConvOnet).  Tolerances: the Gaussian Fourier embedding feeds sin() arguments of
several hundred radians, so one ulp of the argument is ~3e-5 absolute in the embedding;
fp32 oracle vs fp32 kernel agree to ~1e-4 on outputs (stated per assert)."""
import numpy as np
import pytest
import torch

from helpers import max_abs, rel_err

BOUND = np.array([[-2.0, 2.0], [-2.0, 2.0], [-2.0, 2.0]])


def nice_pair(device, seed=0, grid_amp=30.0, bound=BOUND, coarse=False, b_scale=0.2):
    import warnings
    from oracle.nice import NiceOracle
    from xrdslam_b200.camera import Camera
    from xrdslam_b200.conv_onet import ConvOnetConfig
    # nn.Linear and xavier_uniform_ draw from the global generator: seed it, locally
    with torch.random.fork_rng():
        torch.manual_seed(seed)
        ora = NiceOracle(bound, seed=seed, coarse=coarse)
    g = torch.Generator().manual_seed(seed + 5)
    with torch.no_grad():
        for k in ora.grids:
            ora.grids[k].mul_(grid_amp)
        for dec in (ora.middle, ora.fine, ora.color):
            dec.B.mul_(b_scale)  # 0.2: keeps sin() arguments moderate for a tight comparison
            for lin in list(dec.fc_c) + list(dec.pts) + [dec.out]:
                lin.bias.copy_(torch.randn(lin.bias.shape, generator=g) * 0.1)
        if coarse:
            for lin in list(ora.coarse.pts) + [ora.coarse.out]:
                lin.bias.copy_(torch.randn(lin.bias.shape, generator=g) * 0.1)
    with warnings.catch_warnings():
        # no pretrained checkpoints in the tests
        warnings.filterwarnings('ignore', message='ConvOnet: no pretrained checkpoint',
                                category=RuntimeWarning)
        model = ConvOnetConfig(coarse=coarse, mapping_frustum_feature_selection=False).setup(
            camera=Camera(320., 320., 319.5, 239.5, 640, 480), bounding_box=bound)
    with torch.no_grad():
        for name in ('middle', 'fine', 'color'):
            o = getattr(ora, name)
            m = getattr(model.decoder, name + '_decoder')
            m.embedder._B.copy_(o.B)
            for i in range(5):
                m.fc_c[i].weight.copy_(o.fc_c[i].weight); m.fc_c[i].bias.copy_(o.fc_c[i].bias)
                m.pts_linears[i].weight.copy_(o.pts[i].weight)
                m.pts_linears[i].bias.copy_(o.pts[i].bias)
            m.output_linear.weight.copy_(o.out.weight); m.output_linear.bias.copy_(o.out.bias)
        if coarse:
            m = model.decoder.coarse_decoder
            for i in range(5):
                m.pts_linears[i].weight.copy_(ora.coarse.pts[i].weight)
                m.pts_linears[i].bias.copy_(ora.coarse.pts[i].bias)
            m.output_linear.weight.copy_(ora.coarse.out.weight)
            m.output_linear.bias.copy_(ora.coarse.out.bias)
        for k in ora.grids:
            model.set_grid(k, ora.grids[k])
    assert torch.equal(model.bounding_box, ora.bound)
    model.to(device)
    return ora, model


def rays(R, seed):
    g = torch.Generator().manual_seed(seed)
    rays_o = (torch.rand(R, 3, generator=g) - 0.5) * 0.6
    rays_d = torch.nn.functional.normalize(torch.randn(R, 3, generator=g), dim=-1)
    td = torch.rand(R, 1, generator=g) * 1.5 + 0.3
    td[3::7] = 0
    ts = torch.rand(R, 3, generator=g)
    return rays_o, rays_d, ts, td


@pytest.mark.gpu
@pytest.mark.parametrize('stage', ['middle', 'fine', 'color'])
@pytest.mark.parametrize('is_mapping', [True, False])
def test_nice_step_parity(cuda_dev, stage, is_mapping):
    ora, model = nice_pair(cuda_dev)
    R = 200
    rays_o, rays_d, ts, td = rays(R, 11)
    rays_o.requires_grad_(True)
    rays_d.requires_grad_(True)
    out_o, ld_o, tot_o = ora.step(rays_o, rays_d, ts, td, is_mapping, stage)
    tot_o.backward()
    ro = rays_o.detach().to(cuda_dev).requires_grad_(True)
    rd = rays_d.detach().to(cuda_dev).requires_grad_(True)
    inp = dict(rays_o=ro, rays_d=rd, target_s=ts.to(cuda_dev), target_d=td.to(cuda_dev),
               stage=stage, is_mapping=is_mapping)
    out = model(inp)
    ld = model.get_loss_dict(out, inp, is_mapping, stage)
    assert set(ld) == set(ld_o)
    sum(ld.values()).backward()
    torch.cuda.synchronize()
    assert max_abs(out['depth'], out_o['depth']) < 2e-4
    assert max_abs(out['uncertainty'], out_o['uncertainty']) < 2e-4
    assert max_abs(out['rgb'], out_o['rgb']) < 2e-4
    for k in ld_o:
        a, b = float(ld[k].detach()), float(ld_o[k].detach())
        assert abs(a - b) <= 2e-4 * max(abs(b), 1.0), (k, a, b)
    names = ['grid_middle'] + (['grid_fine'] if stage != 'middle' else []) + \
        (['grid_color'] if stage == 'color' else [])
    for k in names:
        g_o = ora.grids[k].grad.squeeze(0).permute(1, 2, 3, 0)
        assert rel_err(model.grids[k].grad, g_o) < 2e-3, k
    assert rel_err(ro.grad, rays_o.grad) < 5e-3
    assert rel_err(rd.grad, rays_d.grad) < 5e-3
    if stage == 'color':
        m, o = model.decoder.color_decoder, ora.color
        assert rel_err(m.embedder._B.grad, o.B.grad) < 5e-3
        for i in range(5):
            assert rel_err(m.pts_linears[i].weight.grad, o.pts[i].weight.grad) < 2e-3, i
            assert rel_err(m.pts_linears[i].bias.grad, o.pts[i].bias.grad) < 2e-3, i
            assert rel_err(m.fc_c[i].weight.grad, o.fc_c[i].weight.grad) < 2e-3, i
            assert rel_err(m.fc_c[i].bias.grad, o.fc_c[i].bias.grad) < 2e-3, i
        assert rel_err(m.output_linear.weight.grad[:3], o.out.weight.grad[:3]) < 2e-3
        assert rel_err(m.output_linear.bias.grad[:3], o.out.bias.grad[:3]) < 2e-3


@pytest.mark.gpu
def test_nice_z_vals_bit_exact(cuda_dev):
    """float64 sample depths (far from the bound, surface band, sort) are bit-exact."""
    import ctypes as C
    from xrdslam_b200 import _cabi
    ora, model = nice_pair(cuda_dev)
    R = 333
    rays_o, rays_d, ts, td = rays(R, 5)
    z_o = ora.sample_z(rays_o, rays_d, td)
    # run forward-only with z output requested through the raw C-ABI
    dev = cuda_dev
    o, _ = model._launch('middle', True, rays_o.to(dev), rays_d.to(dev), None, td.to(dev), False)
    # z_vals are internal unless requested: call again capturing them
    z = torch.empty(R, 48, dtype=torch.float64, device=dev)
    model._z_capture = z
    o2, _ = model._launch('middle', True, rays_o.to(dev), rays_d.to(dev), None, td.to(dev), False)
    assert torch.equal(z.cpu(), z_o)


def test_nice_shapes_match_survey_q2():
    """Default office0 bound -> middle 31x37x35, fine/color 63x75x71 (Z,Y,X)."""
    from xrdslam_b200.camera import Camera
    from xrdslam_b200.conv_onet import ConvOnetConfig
    m = ConvOnetConfig().setup(camera=Camera(320., 320., 319.5, 239.5, 640, 480),
                               bounding_box=np.array([[-5.5, 5.9], [-6.7, 5.4], [-4.7, 5.3]]))
    assert tuple(m.grids['grid_middle'].shape) == (31, 37, 35, 32)
    assert tuple(m.grids['grid_fine'].shape) == (63, 75, 71, 32)
    assert tuple(m.grid_c['grid_color'].shape) == (1, 32, 63, 75, 71)


@pytest.mark.gpu
@pytest.mark.parametrize('tag,is_mapping', [('map', True), ('trk', False)])
def test_nice_cuda_matches_reference_golden(cuda_dev, tag, is_mapping):
    """CUDA path vs vectors produced by the reference's own ConvOnet class."""
    from helpers import load_golden_nice, nice_from_golden
    g = load_golden_nice()
    model = nice_from_golden(g, 'model', cuda_dev)
    t = lambda k: torch.from_numpy(g[k]).to(cuda_dev)
    ro = t('rays_o').requires_grad_(True)
    rd = t('rays_d').requires_grad_(True)
    inp = dict(rays_o=ro, rays_d=rd, target_s=t('target_s'), target_d=t('target_d'),
               stage='color', is_mapping=is_mapping)
    out = model(inp)
    ld = model.get_loss_dict(out, inp, is_mapping, 'color')
    sum(ld.values()).backward()
    assert np.abs(out['rgb'].cpu().numpy() - g[tag + '.rgb']).max() < 2e-4
    assert np.abs(out['depth'].cpu().numpy() - g[tag + '.depth']).max() < 2e-4
    got = np.array([float(ld['depth_loss'].detach()), float(ld['rgb_loss'].detach())])
    assert np.allclose(got, g[tag + '.losses'], rtol=2e-4)
    assert rel_err(ro.grad, torch.from_numpy(g[tag + '.d_rays_o'])) < 5e-3
    assert rel_err(rd.grad, torch.from_numpy(g[tag + '.d_rays_d'])) < 5e-3
    cd = model.decoder.color_decoder
    assert rel_err(cd.embedder._B.grad, torch.from_numpy(g[tag + '.d_B'])) < 5e-3
    assert rel_err(cd.pts_linears[3].weight.grad, torch.from_numpy(g[tag + '.d_pts3_w'])) < 2e-3
    assert rel_err(cd.fc_c[0].weight.grad, torch.from_numpy(g[tag + '.d_fcc0_w'])) < 2e-3
    gc = model.grid_c['grid_color'].grad if False else model.grids['grid_color'].grad
    gc_ref_layout = gc.permute(3, 0, 1, 2)
    assert abs(float(gc.double().norm()) - float(g[tag + '.d_grid_color_norm'])) \
        <= 2e-3 * float(g[tag + '.d_grid_color_norm'])
    assert rel_err(gc_ref_layout[:, 10:14, 10:14, 10:14],
                   torch.from_numpy(g[tag + '.d_grid_color_slice'])) < 2e-3


@pytest.mark.gpu
def test_nice_coarse_stage_parity(cuda_dev):
    """Stage 'coarse' (reference default coarse=True: MLP_no_xyz on the 2 m grid over the doubled
    bound, 32 uniform samples without depth guidance, mapping depth loss) against
    oracle/nice.py, itself bit-identical to the reference ConvOnet(coarse=True)
    (tests/test_oracle_cpu.py::test_nice_oracle_coarse_stage_matches_reference_class_live)."""
    import warnings
    from oracle.nice import NiceOracle
    from xrdslam_b200.camera import Camera
    from xrdslam_b200.conv_onet import ConvOnetConfig
    ora = NiceOracle(BOUND, seed=2, coarse=True)
    g = torch.Generator().manual_seed(9)
    with torch.no_grad():
        ora.grids['grid_coarse'].mul_(60.0)
        for lin in list(ora.coarse.pts) + [ora.coarse.out]:
            lin.bias.copy_(torch.randn(lin.bias.shape, generator=g) * 0.1)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore', RuntimeWarning)  # no pretrained checkpoints in the tests
        model = ConvOnetConfig(coarse=True, mapping_frustum_feature_selection=False).setup(
            camera=Camera(320., 320., 319.5, 239.5, 640, 480), bounding_box=BOUND)
    assert tuple(model.grid_c['grid_coarse'].shape) == tuple(ora.grids['grid_coarse'].shape)
    with torch.no_grad():
        m = model.decoder.coarse_decoder
        for i in range(5):
            m.pts_linears[i].weight.copy_(ora.coarse.pts[i].weight)
            m.pts_linears[i].bias.copy_(ora.coarse.pts[i].bias)
        m.output_linear.weight.copy_(ora.coarse.out.weight)
        m.output_linear.bias.copy_(ora.coarse.out.bias)
        model.set_grid('grid_coarse', ora.grids['grid_coarse'])
    model.to(cuda_dev)
    R = 333
    rays_o, rays_d, ts, td = rays(R, 31)
    rays_o.requires_grad_(True)
    rays_d.requires_grad_(True)
    out_o, ld_o, tot_o = ora.step(rays_o, rays_d, ts, td, True, 'coarse')
    tot_o.backward()
    ro = rays_o.detach().to(cuda_dev).requires_grad_(True)
    rd = rays_d.detach().to(cuda_dev).requires_grad_(True)
    z = torch.empty(R, 32, dtype=torch.float64, device=cuda_dev)
    model._z_capture = z
    inp = dict(rays_o=ro, rays_d=rd, target_s=ts.to(cuda_dev), target_d=td.to(cuda_dev),
               stage='coarse', is_mapping=True)
    out = model(inp)
    ld = model.get_loss_dict(out, inp, True, 'coarse')
    assert set(ld) == set(ld_o) == {'depth_loss'}
    sum(ld.values()).backward()
    torch.cuda.synchronize()
    assert torch.equal(z.cpu(), out_o['z_vals'])            # f64 sample depths: bit-exact
    assert max_abs(out['depth'], out_o['depth']) < 2e-4
    assert max_abs(out['uncertainty'], out_o['uncertainty']) < 2e-4
    a, b = float(ld['depth_loss'].detach()), float(ld_o['depth_loss'].detach())
    assert abs(a - b) <= 2e-4 * max(abs(b), 1.0)
    g_o = ora.grids['grid_coarse'].grad.squeeze(0).permute(1, 2, 3, 0)
    assert rel_err(model.grids['grid_coarse'].grad, g_o) < 2e-3
    assert rel_err(ro.grad, rays_o.grad) < 5e-3
    assert rel_err(rd.grad, rays_d.grad) < 5e-3
    # forward-only (render_img) path returns the same maps
    with torch.no_grad():
        o2 = model(dict(rays_o=ro.detach(), rays_d=rd.detach(), target_s=None,
                        target_d=td.to(cuda_dev), stage='coarse'))
    assert torch.equal(o2['depth'], out['depth'])


@pytest.mark.gpu
def test_nice_mesher_queries_match_oracle(cuda_dev):
    """ConvOnet.query_fn / color_func (mesher path, conv_onet.py:213-240) == the oracle's
    NICE.forward restatement at free points, inside and outside the bound."""
    ora, model = nice_pair(cuda_dev)
    g = torch.Generator().manual_seed(4)
    pts = (torch.rand(2500, 3, generator=g) - 0.5) * 4.6  # some outside [-2, 2]^3 (border clamp)
    with torch.no_grad():
        fine_o = ora.decode(pts, 'fine')
        col_o = ora.decode(pts, 'color')
    fine = model.query_fn(pts.to(cuda_dev))
    col = model.color_func(pts.to(cuda_dev))
    assert fine.shape == (2500, 4) and col.shape == (2500, 4)
    assert max_abs(fine, fine_o) < 2e-4
    assert max_abs(col, col_o) < 2e-4
