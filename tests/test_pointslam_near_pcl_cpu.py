"""Point-SLAM rendering_sample_near_pcl on the CPU: the restatement in
oracle/pointslam_near_pcl.py against numpy's linspace, the second-hit rule, and the reference's
own NeuralPointCloud.sample_near_pcl / render_batch_ray (tests/golden/pointslam_near_pcl.npz,
and live where the reference is available)."""
import os

import numpy as np
import pytest
import torch

from helpers import load_golden_pointslam, max_abs, pointslam_from_golden, rel_err
from oracle import pointslam_near_pcl as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden',
                      'pointslam_near_pcl.npz')


def load_golden():
    g = np.load(GOLDEN)
    return {k: g[k] for k in g.files}


def bits(a):
    a = np.ascontiguousarray(np.asarray(a))
    return a.view(np.int32 if a.dtype == np.float32 else np.int64)


def near_oracle(g):
    """NearPclOracle with the decoders and cloud of pointslam_geo_step.npz."""
    base = pointslam_from_golden(g, 'oracle')
    ora = O.NearPclOracle()
    ora.geo.load_state_dict(base.geo.state_dict())
    ora.col.load_state_dict(base.col.state_dict())
    ora.set_cloud(base.cloud, base.geo_feats.detach(), col_feats=base.col_feats.detach())
    return ora


def test_linspace_f64_is_numpy_linspace():
    rng = np.random.default_rng(0)
    cases = [(0.3, 2.4), (2.4, 0.3), (0.3, 0.3), (1.0, 1.0 + 1e-300), (0.0, 5e-324),
             (-1.5, 7.25), (0.3, float(np.float32(3.1)))]
    cases += [tuple(rng.uniform(-2, 12, 2)) for _ in range(500)]
    for a, b in cases:
        for n in (2, 3, 5, 16, 25):
            assert np.array_equal(bits(O.linspace_f64(a, b, n)), bits(np.linspace(a, b, n))), (a, b, n)


def test_linspace_f32_formula():
    """torch's two-sided formula: start + step k below n / 2, end - step (n - 1 - k) above."""
    z = O.linspace_f32(0.3, np.float32(2.4), 25)
    step = np.float32((np.float32(2.4) - np.float32(0.3)) / np.float32(24))
    assert z[0] == np.float32(0.3) and z[-1] == np.float32(2.4)
    assert z[5] == np.float32(0.3) + step * np.float32(5)
    assert z[20] == np.float32(2.4) - step * np.float32(4)


def _cloud_at(ro, rd, zq, ks):
    """One cloud point on the ray at each march index in ks."""
    return torch.stack([ro + rd * float(zq[k]) for k in ks])


@pytest.mark.parametrize('ks', [[], [6], [3, 7], [3, 7, 12], [23, 24], [0, 1, 2, 3, 24]])
def test_second_hit_rule(ks):
    """z runs from the first to the SECOND hit (the reference's item[1]), not to the last."""
    far = torch.tensor(2.4)
    ro, rd = torch.zeros(3), torch.tensor([0.0, 0.0, 1.0])
    zq = O.linspace_f32(0.3, np.float32(2.4), O.MARCH)
    cloud = _cloud_at(ro, rd, zq, ks) if ks else torch.zeros(0, 3)
    z, near = O.sample_near_pcl(cloud, ro[None], rd[None], torch.zeros(1), far, 0.3, 5, 0.08)
    sec = np.linspace(0.3, float(np.float32(2.4)), 25)
    if len(ks) >= 2:
        assert near.item()
        want = np.linspace(sec[ks[0]], sec[ks[1]], 5)
    else:
        assert not near.item()
        want = np.linspace(0.3, float(np.float32(2.4)), 5)
    assert np.array_equal(bits(z[0].numpy()), bits(want.astype(np.float32)))


def test_rays_with_depth_are_left_alone():
    z, near = O.sample_near_pcl(torch.zeros(0, 3), torch.zeros(3, 3), torch.eye(3),
                                torch.tensor([1.0, 0.0, float('nan')]), torch.tensor(2.0), 0.3, 5,
                                0.08)
    assert near.tolist() == [True, False, False] and (z[0] == 0).all()


def test_oracle_sampler_matches_reference_golden():
    n = load_golden()
    cloud = torch.from_numpy(load_golden_pointslam()['cloud_pos'])
    ro, rd = torch.from_numpy(n['s.rays_o']), torch.from_numpy(n['s.rays_d'])
    for i in range(2):
        z, near = O.sample_near_pcl(cloud, ro, rd, torch.zeros(ro.shape[0]),
                                    torch.from_numpy(n[f's{i}.far']), 0.3, 5, 0.08)
        assert np.array_equal(bits(z.numpy()), bits(n[f's{i}.z']))
        assert np.array_equal(~near.numpy(), n[f's{i}.invalid'])
        assert 0 < n[f's{i}.invalid'].sum() < ro.shape[0]


@pytest.mark.parametrize('stage', ['geometry', 'color'])
@pytest.mark.parametrize('tag,is_mapping', [('map', True), ('trk', False)])
def test_oracle_render_matches_reference_golden(stage, tag, is_mapping):
    """render_batch_ray with the option on: z and masks bit for bit; depth, colour, losses and
    gradients at the gates of the option-off oracle tests."""
    g, n = load_golden_pointslam(), load_golden()
    key = stage[0] + tag
    ora = near_oracle(g)
    ro = torch.from_numpy(g['rays_o']).requires_grad_(True)
    rd = torch.from_numpy(g['rays_d']).requires_grad_(True)
    td = torch.from_numpy(n['r.target_d'])
    ts = torch.from_numpy(g['target_s']) if stage == 'color' else torch.zeros(td.shape[0], 3)
    out = ora.render(ro, rd, td, torch.from_numpy(g['radius']), torch.from_numpy(g['rand_feat']),
                     stage, torch.from_numpy(g['rand_feat_color']))
    ld = ora.loss_dict(out, td, ts, is_mapping)
    (sum(ld.values()) if stage == 'color' else ld['geo_loss']).backward()
    Z = n[key + '.zero_rays']
    assert np.array_equal(bits(out['z_vals'].detach().numpy()[Z]), bits(n[key + '.z_zero']))
    assert np.array_equal(~ora._near_pcl[1].numpy()[Z], n[key + '.invalid_zero'])
    assert np.array_equal(out['valid_ray_mask'].numpy(), n[key + '.valid'])
    assert (out['depth'].detach()[Z] != 0).any()  # zero-depth rays keep their depth
    assert max_abs(out['depth'], n[key + '.depth']) < 1e-6
    assert max_abs(out['uncertainty'], n[key + '.uncertainty']) < 1e-6
    assert max_abs(out['rgb'], n[key + '.rgb']) < 1e-5
    for i, v in enumerate(ld.values()):
        ref = float(n[key + '.losses'][i])
        assert abs(float(v.detach()) - ref) < 1e-4 * max(1, abs(ref))
    assert rel_err(ora.geo_feats.grad, n[key + '.d_geo_feats']) < 1e-4
    assert rel_err(ro.grad, n[key + '.d_rays_o']) < 1e-3
    assert rel_err(rd.grad, n[key + '.d_rays_d']) < 1e-3
    if stage == 'color':
        assert rel_err(ora.col_feats.grad, n[key + '.d_col_feats']) < 1e-4


def test_oracle_render_without_depth_matches_reference_golden():
    g, n = load_golden_pointslam(), load_golden()
    ora = near_oracle(g)
    with torch.no_grad():
        out = ora.render(torch.from_numpy(g['rays_o']), torch.from_numpy(g['rays_d']), None,
                         torch.from_numpy(g['radius']), torch.from_numpy(g['rand_feat']), 'color',
                         torch.from_numpy(g['rand_feat_color']))
    assert np.array_equal(bits(out['z_vals'].numpy()), bits(n['nodepth.z']))
    assert np.array_equal(out['valid_ray_mask'].numpy(), n['nodepth.valid'])
    assert max_abs(out['depth'], n['nodepth.depth']) < 1e-6
    assert max_abs(out['rgb'], n['nodepth.rgb']) < 1e-5


@pytest.mark.needs_reference
def test_golden_is_what_the_reference_computes():
    """The reference's own sample_near_pcl, live, equals the golden and the oracle."""
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))
    import make_golden_near_pcl as M
    g, n = load_golden_pointslam(), load_golden()
    ref = M.reference_model(g)
    ro, rd = torch.from_numpy(n['s.rays_o']), torch.from_numpy(n['s.rays_d'])
    cloud = torch.from_numpy(g['cloud_pos'])
    for far in (2.4, 3.1, 10.0):
        far_t = torch.tensor(far)
        z, invalid = ref.neural_point_cloud.sample_near_pcl(ro.clone(), rd.clone(), 0.3, far_t, 5)
        zo, near = O.sample_near_pcl(cloud, ro, rd, torch.zeros(ro.shape[0]), far_t, 0.3, 5, 0.08)
        assert np.array_equal(bits(z.numpy()), bits(zo.numpy()))
        assert torch.equal(invalid, ~near)
    z, invalid = ref.neural_point_cloud.sample_near_pcl(ro.clone(), rd.clone(), 0.3,
                                                        torch.from_numpy(n['s0.far']), 5)
    assert np.array_equal(bits(z.numpy()), bits(n['s0.z']))
    with torch.no_grad():
        torch.manual_seed(777)
        out = ref.render_batch_ray(torch.from_numpy(g['rays_d']), torch.from_numpy(g['rays_o']),
                                   'color', gt_depth=None,
                                   dynamic_r_query=torch.from_numpy(g['radius']))
    assert torch.equal(out['valid_ray_mask'], torch.from_numpy(n['nodepth.valid']))
    assert torch.equal(out['depth'], torch.from_numpy(n['nodepth.depth']))
