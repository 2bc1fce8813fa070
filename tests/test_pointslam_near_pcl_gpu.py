"""Point-SLAM rendering_sample_near_pcl on the device: xrd_pointslam_sample_near_pcl bit for bit
against oracle/pointslam_near_pcl.py and the reference golden (tests/golden/pointslam_near_pcl.npz),
the step with the option on against the oracle and the golden, render_img with holes, and a run
through the command line."""
import os

import numpy as np
import pytest
import torch

from helpers import load_golden_pointslam, max_abs, pointslam_from_golden, rel_err
from oracle import pointslam_near_pcl as O
from test_pointslam_near_pcl_cpu import bits, load_golden, near_oracle

pytestmark = pytest.mark.gpu


def _model(g, dev, **cfg):
    model = pointslam_from_golden(g, 'b200', dev)
    model.config.rendering_sample_near_pcl = True
    for k, v in cfg.items():
        setattr(model.config, k, v)
    return model


def _sample(npc, ro, rd, td, far, dev):
    f = lambda t: t.to(dev, torch.float32).contiguous()
    z, near = npc.near_pcl_samples(f(ro), f(rd), f(td.reshape(-1)), f(far.reshape(1)), 0.3, 5)
    return z.cpu(), near.cpu().bool()


def _check(npc, cloud, ro, rd, td, far, dev):
    z, near = _sample(npc, ro, rd, td, far, dev)
    zo, nearo = O.sample_near_pcl(cloud, ro, rd, td, far, 0.3, 5, 0.08)
    Z = ~(td.reshape(-1) > 0)
    assert torch.equal(near, nearo)
    assert np.array_equal(bits(z[Z].numpy()), bits(zo[Z].numpy()))
    return z, near


def test_sampler_matches_reference_golden(cuda_dev):
    g, n = load_golden_pointslam(), load_golden()
    npc = pointslam_from_golden(g, 'b200', cuda_dev).neural_point_cloud
    ro, rd = torch.from_numpy(n['s.rays_o']), torch.from_numpy(n['s.rays_d'])
    for i in range(2):
        far = torch.from_numpy(n[f's{i}.far'])
        z, invalid = npc.sample_near_pcl(ro, rd, 0.3, far, 5)
        assert np.array_equal(bits(z.cpu().numpy()), bits(n[f's{i}.z']))
        assert np.array_equal(invalid.cpu().numpy(), n[f's{i}.invalid'])
        _check(npc, torch.from_numpy(g['cloud_pos']), ro, rd, torch.zeros(ro.shape[0]), far,
               cuda_dev)


def test_sampler_hit_patterns(cuda_dev):
    """0, 1, 2 and many hits, hits only at the last two march points, NaN and positive depth
    between them, and an empty cloud."""
    from xrdslam_b200.neural_point_cloud import NeuralPointCloud
    far = torch.tensor(2.4)
    zq = O.linspace_f32(0.3, np.float32(2.4), O.MARCH)
    patterns = [[], [6], [3, 7], [3, 7, 12], [23, 24], [0, 1, 2, 3, 24], list(range(25))]
    ro = torch.tensor([[0.0, 0.0, 0.0]]).repeat(len(patterns), 1)
    ro[:, 0] = torch.arange(len(patterns)) * 1.0  # rays 1 m apart: separate hit sets
    rd = torch.tensor([[0.0, 0.0, 1.0]]).repeat(len(patterns), 1)
    pts = [ro[i] + rd[i] * float(zq[k]) for i, ks in enumerate(patterns) for k in ks]
    cloud = torch.stack(pts)
    npc = NeuralPointCloud(device=cuda_dev)
    npc.set_cloud(cloud, torch.zeros(cloud.shape[0], 32))
    td = torch.zeros(len(patterns))
    z, near = _check(npc, cloud, ro, rd, td, far, cuda_dev)
    assert near.tolist() == [len(p) >= 2 for p in patterns]
    sec = np.linspace(0.3, float(np.float32(2.4)), 25)
    assert np.array_equal(bits(z[4].numpy()), bits(np.linspace(sec[23], sec[24], 5).astype(np.float32)))
    # depth on some rays (left alone, near = 1), NaN on others (sampled)
    td2 = torch.tensor([1.0, float('nan'), 0.0, 2.0, float('nan'), -1.0, 0.5])
    _, near2 = _check(npc, cloud, ro, rd, td2, far, cuda_dev)
    assert near2[0] and near2[3] and near2[6] and not near2[1]
    # empty cloud: every zero-depth ray is invalid with np.linspace(near_end, far, 5)
    empty = NeuralPointCloud(device=cuda_dev)
    z, invalid = empty.sample_near_pcl(ro, rd, 0.3, far, 5)
    assert invalid.all()
    want = np.linspace(0.3, float(np.float32(2.4)), 5).astype(np.float32)
    assert np.array_equal(bits(z.cpu().numpy()), bits(np.tile(want, (len(patterns), 1))))


def _inputs(g, td, dev, stage, is_mapping=None, grads=True):
    ro = torch.from_numpy(g['rays_o']).to(dev).requires_grad_(grads)
    rd = torch.from_numpy(g['rays_d']).to(dev).requires_grad_(grads)
    ts = torch.from_numpy(g['target_s']).to(dev) if stage == 'color' else \
        torch.zeros(ro.shape[0], 3, device=dev)
    inp = dict(rays_o=ro, rays_d=rd, target_d=td.to(dev), target_s=ts, stage=stage,
               batch_dynamic_r=torch.from_numpy(g['radius']).to(dev),
               rand_feat=torch.from_numpy(g['rand_feat']).to(dev),
               rand_feat_color=torch.from_numpy(g['rand_feat_color']).to(dev))
    if is_mapping is not None:
        inp['is_mapping'] = is_mapping
    return inp, ro, rd


def _run(model, g, td, dev, stage, is_mapping):
    inp, ro, rd = _inputs(g, td, dev, stage, is_mapping)
    R, S = ro.shape[0], model.config.rendering_n_surface
    model._z_capture = torch.empty(R, S, device=dev)
    npc = model.neural_point_cloud
    for t in [npc.geo_feats, npc.col_feats] + list(model.decoder.parameters()):
        t.grad = None
    out = model(inp)
    ld = model.get_loss_dict(out, inp, is_mapping)
    (sum(ld.values()) if stage == 'color' else ld['geo_loss']).backward()
    z = model._z_capture.cpu()
    del model._z_capture
    return out, ld, ro, rd, z


@pytest.mark.parametrize('stage', ['geometry', 'color'])
@pytest.mark.parametrize('tag,is_mapping', [('map', True), ('trk', False)])
def test_step_matches_reference_golden(cuda_dev, stage, tag, is_mapping):
    g, n = load_golden_pointslam(), load_golden()
    key = stage[0] + tag
    model = _model(g, cuda_dev)
    td = torch.from_numpy(n['r.target_d'])
    out, ld, ro, rd, z = _run(model, g, td, cuda_dev, stage, is_mapping)
    Z = n[key + '.zero_rays']
    assert np.array_equal(bits(z.numpy()[Z]), bits(n[key + '.z_zero']))
    assert np.array_equal(out['valid_ray_mask'].cpu().numpy(), n[key + '.valid'])
    assert max_abs(out['depth'], n[key + '.depth']) < 2e-5
    assert max_abs(out['uncertainty'], n[key + '.uncertainty']) < 1e-6
    tol = 1e-3 if stage == 'color' else 2e-4
    for i, v in enumerate(ld.values()):
        ref = float(n[key + '.losses'][i])
        assert abs(float(v.detach()) - ref) < 2e-4 * max(1, abs(ref))
    npc = model.neural_point_cloud
    assert rel_err(npc.geo_feats.grad, n[key + '.d_geo_feats']) < tol
    assert rel_err(ro.grad, n[key + '.d_rays_o']) < 5 * tol
    assert rel_err(rd.grad, n[key + '.d_rays_d']) < 5 * tol
    if stage == 'color':
        assert max_abs(out['rgb'], n[key + '.rgb']) < 2e-5
        assert rel_err(npc.col_feats.grad, n[key + '.d_col_feats']) < tol


@pytest.mark.parametrize('handle_dynamic', [True, False])
@pytest.mark.parametrize('stage', ['geometry', 'color'])
@pytest.mark.parametrize('is_mapping', [True, False])
def test_step_matches_oracle(cuda_dev, stage, is_mapping, handle_dynamic):
    """Holes with zero and negative depth: z bit for bit, the rest at the option-off gates."""
    g = load_golden_pointslam()
    model = _model(g, cuda_dev, tracking_handle_dynamic=handle_dynamic)
    td = torch.from_numpy(g['target_d']).clone().reshape(-1, 1)
    td[1::3] = 0
    td[4] = -0.5
    out, ld, ro, rd, z = _run(model, g, td, cuda_dev, stage, is_mapping)
    ora = near_oracle(g)
    ro_o = torch.from_numpy(g['rays_o']).requires_grad_(True)
    rd_o = torch.from_numpy(g['rays_d']).requires_grad_(True)
    ts = torch.from_numpy(g['target_s']) if stage == 'color' else torch.zeros(td.shape[0], 3)
    out_o = ora.render(ro_o, rd_o, td, torch.from_numpy(g['radius']),
                       torch.from_numpy(g['rand_feat']), stage,
                       torch.from_numpy(g['rand_feat_color']))
    ld_o = ora.loss_dict(out_o, td, ts, is_mapping, handle_dynamic)
    (sum(ld_o.values()) if stage == 'color' else ld_o['geo_loss']).backward()
    assert np.array_equal(bits(z.numpy()), bits(out_o['z_vals'].detach().numpy()))
    assert torch.equal(out['valid_ray_mask'].cpu(), out_o['valid_ray_mask'])
    assert max_abs(out['depth'], out_o['depth']) < 2e-5
    assert max_abs(out['uncertainty'], out_o['uncertainty']) < 1e-6
    for k in ld_o:
        ref = float(ld_o[k].detach())
        assert abs(float(ld[k].detach()) - ref) < 2e-4 * max(1, abs(ref)), k
    npc = model.neural_point_cloud
    tol = 1e-3 if stage == 'color' else 2e-4
    assert rel_err(npc.geo_feats.grad, ora.geo_feats.grad) < tol
    assert rel_err(ro.grad, ro_o.grad) < 5 * tol
    assert rel_err(rd.grad, rd_o.grad) < 5 * tol


def test_tracking_mask_moves_with_zero_depth_residuals(cuda_dev):
    """With depth zeroed, every hole adds tmp = 0 to the tracking median; with the option on it
    adds its real residual, so the median, the mask and the loss change."""
    g = load_golden_pointslam()
    td = torch.from_numpy(g['target_d']).clone().reshape(-1, 1)
    td[::2] = 0  # half the rays: the option-off median is 0 and the mask empty
    losses = {}
    for on in (False, True):
        model = _model(g, cuda_dev, rendering_sample_near_pcl=on)
        out, ld, _, _, _ = _run(model, g, td, cuda_dev, 'geometry', False)
        losses[on] = float(ld['geo_loss'].detach())
    ora = near_oracle(g)
    out_o = ora.render(torch.from_numpy(g['rays_o']), torch.from_numpy(g['rays_d']), td,
                       torch.from_numpy(g['radius']), torch.from_numpy(g['rand_feat']))
    ref = float(ora.loss_dict(out_o, td, torch.zeros(td.shape[0], 3), False)['geo_loss'].detach())
    assert losses[False] == 0.0 and ref > 0
    assert abs(losses[True] - ref) < 2e-4 * max(1, ref)


def test_render_without_depth(cuda_dev):
    """gt_depth None: every ray is sampled near the cloud with far = 10."""
    g, n = load_golden_pointslam(), load_golden()
    model = _model(g, cuda_dev)
    inp, _, _ = _inputs(g, torch.zeros(1), cuda_dev, 'color', grads=False)
    inp['target_d'] = None
    R = inp['rays_o'].shape[0]
    model._z_capture = torch.empty(R, 5, device=cuda_dev)
    with torch.no_grad():
        out = model(inp)
    assert np.array_equal(bits(model._z_capture.cpu().numpy()), bits(n['nodepth.z']))
    assert np.array_equal(out['valid_ray_mask'].cpu().numpy(), n['nodepth.valid'])
    assert max_abs(out['depth'], n['nodepth.depth']) < 2e-5
    assert max_abs(out['rgb'], n['nodepth.rgb']) < 2e-5


def test_option_without_holes_is_bit_identical(cuda_dev):
    """Without holes the option changes nothing: outputs bit for bit; the gradients, which
    the kernels accumulate with atomics, to rounding."""
    g = load_golden_pointslam()
    td = torch.from_numpy(g['target_d']).clone().reshape(-1, 1)
    td[td <= 0] = 1.5
    outs = []
    for on in (False, True):
        model = _model(g, cuda_dev, rendering_sample_near_pcl=on)
        out, ld, ro, rd, z = _run(model, g, td, cuda_dev, 'color', True)
        outs.append((out['depth'].cpu(), out['rgb'].cpu(), out['valid_ray_mask'].cpu(), z,
                     model.neural_point_cloud.geo_feats.grad.cpu(), rd.grad.cpu()))
    for a, b in zip(outs[0][:4], outs[1][:4]):
        assert torch.equal(a, b)
    for a, b in zip(outs[0][4:], outs[1][4:]):
        assert rel_err(b, a) < 1e-6


def test_render_img_with_holes(cuda_dev):
    """render_img: hole pixels near the cloud get a depth; every other pixel is bit-identical to
    the option-off render."""
    import warnings

    from xrdslam_b200.frame import Frame
    from xrdslam_b200.point_slam import PointSLAMConfig
    from xrdslam_b200.synthetic import make_sequence
    cam, poses, fr = make_sequence(2, width=80, height=60)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore', RuntimeWarning)
        algo = PointSLAMConfig(pixels_adding=2000, mapping_pixels_based_on_color_grad=200).setup(
            camera=cam, device=cuda_dev)
    frames = [Frame(k, fr[k][0], fr[k][1], init_pose=poses[k], separate_LR=True,
                    rot_rep='axis_angle') for k in range(2)]
    np.random.seed(0)
    torch.manual_seed(0)
    for f in frames:
        algo.pre_precessing(f, True)
    depth = fr[1][1].copy()
    depth[10:30, 20:50] = 0
    hole = ~(depth > 0)  # the punched block and the frame's own pixels without depth
    rf = torch.zeros(32, device=cuda_dev)
    res = {}
    for on in (False, True):
        algo.model.config.rendering_sample_near_pcl = on
        res[on] = algo._render_full(poses[1], depth, extra={'stage': 'color', 'rand_feat': rf,
                                                            'rand_feat_color': rf},
                                    per_pixel={'batch_dynamic_r':
                                               algo.dynamic_r_query_allkeyframe['1'].reshape(-1).float()})
    (c0, d0), (c1, d1) = res[False], res[True]
    assert (d0[hole] == 0).all() and (d1[hole] != 0).mean() > 0.5
    assert np.array_equal(d0[~hole], d1[~hole]) and np.array_equal(c0[~hole], c1[~hole])


def test_run_with_option_on_tum_holes(cuda_dev, tmp_path):
    """python -m xrdslam_b200.run point-slam --set model.rendering_sample_near_pcl=True over a
    synthetic TUM folder with holes, then python -m xrdslam_b200.eval scores it."""
    import warnings

    from xrdslam_b200 import run
    from xrdslam_b200 import synthetic as S
    from xrdslam_b200.eval import EvalMatrics
    data, out = str(tmp_path / 'tum'), str(tmp_path / 'out')
    S.write_tum(data, 8, width=224, height=176, turn=0.1)
    sets = dict(tracking_n_iters=10, mapping_n_iters=5, mapping_first_n_iters=30,
                tracking_Wedge=10, tracking_Hedge=10, pixels_adding=800, mapping_sample=500,
                mapping_pixels_based_on_color_grad=200)
    argv = ['point-slam', '--data', data, '--data_type', 'tumrgbd', '--out_dir', out,
            '--device', str(cuda_dev), '--set', 'model.rendering_sample_near_pcl=True']
    for k, v in sets.items():
        argv += ['--set', f'{k}={v!r}']
    torch.manual_seed(0)
    np.random.seed(0)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore', UserWarning)
        warnings.simplefilter('ignore', RuntimeWarning)
        res = run.main(argv)
    assert res['n_frames'] > 0 and os.path.exists(os.path.join(out, 'eval.tar'))
    ev = EvalMatrics(output_dir=out, eval_recon=False, device=str(cuda_dev))
    ev.main()
    assert np.isfinite(float(ev.traj_result['rmse']))
