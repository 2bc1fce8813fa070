"""Parity of the Point-SLAM CUDA path (C-ABI) against oracle/pointslam.py and the golden
fixture generated from the reference's own ConvOnet2 (faiss replaced by exact kNN -- the
contract this framework defines, SURVEY A.4).  Tolerances as in test_nice_gpu.py."""
import numpy as np
import pytest
import torch

from helpers import load_golden_pointslam, max_abs, pointslam_from_golden, rel_err


def _cloud(N, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(N, 3, generator=g) - 0.5) * torch.tensor([2.0, 2.0, 0.3])


@pytest.mark.gpu
@pytest.mark.parametrize('N', [5, 3000, 40000])
def test_knn_exact(cuda_dev, N):
    """Exact 8-NN within the query radius: ids as integer SETS per distance rank (equal
    distances may permute), squared distances bit-exact, sentinels -1 / FLT_MAX."""
    from oracle.pointslam import FLT_MAX, exact_knn
    from xrdslam_b200.neural_point_cloud import NeuralPointCloud
    npc = NeuralPointCloud(device=cuda_dev)
    pos = _cloud(N, 1)
    npc.set_cloud(pos, torch.zeros(N, 32))
    g = torch.Generator().manual_seed(2)
    q = (torch.rand(700, 3, generator=g) - 0.5) * torch.tensor([2.2, 2.2, 0.4])
    q[:50] = pos[torch.arange(50) % N]  # exact hits (D = 0)
    radius = torch.rand(700, generator=g) * 0.12 + 0.02
    D, I, n = npc.find_neighbors(q, radius)
    Do, Io = exact_knn(pos, q, 8)
    r2 = (radius * radius)[:, None]
    inside = Do < r2  # neighbours beyond the radius are not searched (sentinel)
    Do_m = torch.where(inside, Do, torch.full_like(Do, FLT_MAX))
    Io_m = torch.where(inside, Io, torch.full_like(Io, -1))
    assert torch.equal(D.cpu(), Do_m)
    assert torch.equal(n.cpu().long(), inside.sum(1))
    Ic = I.cpu().long()
    same = Ic == Io_m
    # rows where ids differ must be equal-distance permutations
    for r in torch.nonzero(~same.all(1)).flatten().tolist():
        assert sorted(Ic[r].tolist()) == sorted(Io_m[r].tolist()) or \
            torch.equal(Do_m[r], D.cpu()[r])


@pytest.mark.gpu
def test_knn_scalar_radius_and_empty(cuda_dev):
    from xrdslam_b200.neural_point_cloud import NeuralPointCloud
    npc = NeuralPointCloud(device=cuda_dev)
    q = torch.zeros(4, 3)
    D, I, n = npc.find_neighbors(q, 0.1)
    assert (I == -1).all() and (n == 0).all()
    npc.set_cloud(torch.tensor([[0.0, 0.0, 0.05], [1.0, 0, 0]]), torch.zeros(2, 32))
    D, I, n = npc.find_neighbors(q, 0.1)
    assert n.tolist() == [1] * 4 and I[:, 0].tolist() == [0] * 4 and (I[:, 1:] == -1).all()


@pytest.mark.gpu
def test_add_neural_points_matches_reference(cuda_dev):
    """add_neural_points on the golden's first frame reproduces the reference's cloud."""
    from xrdslam_b200.neural_point_cloud import NeuralPointCloud
    g = load_golden_pointslam()
    npc = NeuralPointCloud(device=cuda_dev)
    rd = torch.from_numpy(g['add_rays_d'])
    n = npc.add_neural_points(torch.zeros_like(rd), rd, torch.from_numpy(g['add_depth']),
                              dynamic_radius=torch.full((rd.shape[0],), 0.04))
    assert npc.pts_num() == g['cloud_pos'].shape[0] and n * 3 == npc.pts_num()
    assert max_abs(npc.cloud_pos(), g['cloud_pos']) < 2e-7
    # adding the same frame again adds nothing (every pixel now has a neighbour)
    assert npc.add_neural_points(torch.zeros_like(rd), rd, torch.from_numpy(g['add_depth']),
                                 dynamic_radius=torch.full((rd.shape[0],), 0.04)) == 0


def _run(model, g, is_mapping, dev, grads=True, stage='geometry'):
    ro = torch.from_numpy(g['rays_o']).to(dev).requires_grad_(grads)
    rd = torch.from_numpy(g['rays_d']).to(dev).requires_grad_(grads)
    ts = torch.from_numpy(g['target_s']).to(dev) if 'target_s' in g and stage == 'color' \
        else torch.zeros(ro.shape[0], 3, device=dev)
    inp = dict(rays_o=ro, rays_d=rd, target_d=torch.from_numpy(g['target_d']).to(dev),
               target_s=ts, stage=stage,
               batch_dynamic_r=torch.from_numpy(g['radius']).to(dev), is_mapping=is_mapping)
    for k in ('rand_feat', 'rand_feat_color'):
        if k in g:
            inp[k] = torch.as_tensor(g[k]).to(dev)
    out = model(inp)
    ld = model.get_loss_dict(out, inp, is_mapping)
    if grads:
        npc = model.neural_point_cloud
        for t in [npc.geo_feats, npc.col_feats] + list(model.decoder.parameters()):
            t.grad = None
        (sum(ld.values()) if stage == 'color' else ld['geo_loss']).backward()
    return out, ld, ro, rd


@pytest.mark.gpu
@pytest.mark.parametrize('tag,is_mapping', [('map', True), ('trk', False)])
def test_pointslam_golden(cuda_dev, tag, is_mapping):
    g = load_golden_pointslam()
    model = pointslam_from_golden(g, 'b200', cuda_dev)
    out, ld, ro, rd = _run(model, g, is_mapping, cuda_dev)
    assert torch.equal(out['valid_ray_mask'].cpu(), torch.from_numpy(g[tag + '.valid']))
    assert max_abs(out['depth'], g[tag + '.depth']) < 2e-5
    assert max_abs(out['uncertainty'], g[tag + '.uncertainty']) < 1e-6
    assert abs(float(ld['geo_loss'].detach()) - float(g[tag + '.loss'])) < 2e-4 * max(1, abs(float(g[tag + '.loss'])))
    assert rel_err(model.neural_point_cloud.geo_feats.grad, g[tag + '.d_geo_feats']) < 2e-4
    assert rel_err(ro.grad, g[tag + '.d_rays_o']) < 5e-4
    assert rel_err(rd.grad, g[tag + '.d_rays_d']) < 5e-4


@pytest.mark.gpu
@pytest.mark.parametrize('is_mapping', [True, False])
def test_pointslam_step_vs_oracle(cuda_dev, is_mapping):
    """Bigger seeded case (R = 600 rays, 12k points) incl. rays with no neighbours."""
    from oracle.pointslam import PointOracle
    from xrdslam_b200.camera import Camera
    from xrdslam_b200.conv_onet_pointslam import ConvOnet2Config
    R = 600
    gen = torch.Generator().manual_seed(4)
    rd = torch.nn.functional.normalize(
        torch.randn(R, 3, generator=gen) * torch.tensor([0.4, 0.4, 0.05]) +
        torch.tensor([0, 0, -1.0]), dim=-1)
    d = torch.rand(R, generator=gen) * 0.6 + 1.2
    # cloud: 20 noisy points around each of the first 500 rays' surface points
    surf = (rd * d[:, None])[:500]
    pos = (surf[:, None, :] + torch.randn(500, 24, 3, generator=gen) * 0.03).reshape(-1, 3)
    feats = torch.randn(pos.shape[0], 32, generator=gen) * 0.5
    ora = PointOracle(seed=3)
    with torch.no_grad():
        ora.geo.B.mul_(0.05)
    ora.set_cloud(pos, feats)
    model = ConvOnet2Config().setup(camera=Camera(320., 320., 319.5, 239.5, 640, 480))
    gd = model.decoder.geo_decoder
    with torch.no_grad():
        gd.embedder._B.copy_(ora.geo.B)
        for i in range(5):
            gd.fc_c[i].load_state_dict(ora.geo.fc_c[i].state_dict())
            gd.pts_linears[i].load_state_dict(ora.geo.pts[i].state_dict())
        gd.output_linear.load_state_dict(ora.geo.out.state_dict())
    model.to(cuda_dev)
    model.model_update(cuda_dev).set_cloud(pos, feats)
    td = d.clone().reshape(-1, 1)
    td[7::11] = 0
    radius = torch.rand(R, generator=gen) * 0.06 + 0.04
    rf = torch.randn(32, generator=gen) * 0.01
    # rand_feat (Q6: the feature of sample points without neighbours) is an explicit input on
    # both sides; without it the model draws from the global generator and the comparison
    # depends on which tests ran before
    g = dict(rays_o=np.zeros((R, 3), np.float32), rays_d=rd.numpy(), target_d=td.numpy(),
             radius=radius.numpy(), rand_feat=rf.numpy())
    out, ld, ro, rdg = _run(model, g, is_mapping, cuda_dev)
    ro_o = torch.zeros(R, 3, requires_grad=True)
    rd_o = rd.clone().requires_grad_(True)
    out_o = ora.render(ro_o, rd_o, td, radius, rf)
    l_o = ora.loss(out_o, td, is_mapping)
    l_o.backward()
    assert torch.equal(out['valid_ray_mask'].cpu(), out_o['valid_ray_mask'])
    assert not out_o['valid_ray_mask'].all() and out_o['valid_ray_mask'].any()
    assert max_abs(out['depth'], out_o['depth']) < 2e-5
    assert max_abs(out['uncertainty'], out_o['uncertainty']) < 1e-6
    assert abs(float(ld['geo_loss'].detach()) - float(l_o.detach())) < 2e-4 * max(1.0, abs(float(l_o.detach())))
    assert rel_err(model.neural_point_cloud.geo_feats.grad, ora.geo_feats.grad) < 2e-4
    assert rel_err(ro.grad, ro_o.grad) < 5e-4
    assert rel_err(rdg.grad, rd_o.grad) < 5e-4


@pytest.mark.gpu
@pytest.mark.parametrize('tag,is_mapping', [('cmap', True), ('ctrk', False)])
def test_pointslam_color_golden(cuda_dev, tag, is_mapping):
    """Stage 'color' against the reference ConvOnet2's outputs, losses and every gradient
    (geo/col features, rays, all colour-decoder tensors).  The GEMMs run in the default
    3xTF32 mode (the trunk on mma.sync: P = 400 columns is below the wgmma kernel's 512; the
    neighbour MLP at 8 P = 3200 columns on the wgmma kernel); the softplus
    (beta = 100) trunk amplifies rounding differences ~10x relative to the geometry stage."""
    g = load_golden_pointslam()
    model = pointslam_from_golden(g, 'b200', cuda_dev)
    out, ld, ro, rd = _run(model, g, is_mapping, cuda_dev, stage='color')
    assert max_abs(out['depth'], g[tag + '.depth']) < 2e-5
    assert max_abs(out['rgb'], g[tag + '.rgb']) < 2e-5
    for i, k in enumerate(('geo_loss', 'rgb_loss')):
        ref = float(g[tag + '.losses'][i])
        assert abs(float(ld[k].detach()) - ref) < 2e-4 * max(1, abs(ref)), k
    npc = model.neural_point_cloud
    assert rel_err(npc.geo_feats.grad, g[tag + '.d_geo_feats']) < 1e-3
    assert rel_err(npc.col_feats.grad, g[tag + '.d_col_feats']) < 1e-3
    assert rel_err(ro.grad, g[tag + '.d_rays_o']) < 2e-3
    assert rel_err(rd.grad, g[tag + '.d_rays_d']) < 2e-3
    for k, v in model.decoder.color_decoder.named_parameters():
        assert rel_err(v.grad, g[tag + '.d_cdec.' + k]) < 2e-3, k


@pytest.mark.gpu
@pytest.mark.parametrize('is_mapping', [True, False])
def test_pointslam_color_step_vs_oracle(cuda_dev, is_mapping):
    """Seeded case with R*S not a multiple of 4 (padded columns) and rays without
    neighbours; every gradient against oracle/pointslam.py."""
    from helpers import oracle_cdec_grads
    g = dict(load_golden_pointslam())
    R = 61  # 305 points: exercises the Pp != P padding of the neighbour GEMMs
    for k in ('rays_o', 'rays_d', 'target_d', 'radius', 'target_s'):
        g[k] = g[k][:R].copy()
    g['target_d'][3] = 0  # a zero-depth ray sampled far from the cloud
    g['rays_d'][7] = -g['rays_d'][7]  # a ray that looks away from every point
    model = pointslam_from_golden(g, 'b200', cuda_dev)
    ora = pointslam_from_golden(g, 'oracle')
    out, ld, ro, rd = _run(model, g, is_mapping, cuda_dev, stage='color')
    ro_o = torch.from_numpy(g['rays_o']).requires_grad_(True)
    rd_o = torch.from_numpy(g['rays_d']).requires_grad_(True)
    td, ts = torch.from_numpy(g['target_d']), torch.from_numpy(g['target_s'])
    out_o = ora.render(ro_o, rd_o, td, torch.from_numpy(g['radius']),
                       torch.from_numpy(g['rand_feat']), 'color',
                       torch.from_numpy(g['rand_feat_color']))
    ld_o = ora.loss_dict(out_o, td, ts, is_mapping)
    sum(ld_o.values()).backward()
    assert torch.equal(out['valid_ray_mask'].cpu(), out_o['valid_ray_mask'])
    assert not out_o['valid_ray_mask'].all()
    assert max_abs(out['depth'], out_o['depth']) < 2e-5
    assert max_abs(out['rgb'], out_o['rgb']) < 2e-5
    for k in ld_o:
        ref = float(ld_o[k].detach())
        assert abs(float(ld[k].detach()) - ref) < 2e-4 * max(1, abs(ref)), k
    npc = model.neural_point_cloud
    assert rel_err(npc.geo_feats.grad, ora.geo_feats.grad) < 1e-3
    assert rel_err(npc.col_feats.grad, ora.col_feats.grad) < 1e-3
    assert rel_err(ro.grad, ro_o.grad) < 2e-3
    assert rel_err(rd.grad, rd_o.grad) < 2e-3
    og = oracle_cdec_grads(ora)
    for k, v in model.decoder.color_decoder.named_parameters():
        assert rel_err(v.grad, og[k]) < 2e-3, k


@pytest.mark.gpu
def test_pointslam_color_forward_only_matches_fused(cuda_dev):
    """render_img path (no grad) returns the same colours/depths as the fused step."""
    g = load_golden_pointslam()
    model = pointslam_from_golden(g, 'b200', cuda_dev)
    out, _, _, _ = _run(model, g, True, cuda_dev, stage='color')
    with torch.no_grad():
        inp = dict(rays_o=torch.from_numpy(g['rays_o']).to(cuda_dev),
                   rays_d=torch.from_numpy(g['rays_d']).to(cuda_dev),
                   target_d=torch.from_numpy(g['target_d']).to(cuda_dev), target_s=None,
                   stage='color', batch_dynamic_r=torch.from_numpy(g['radius']).to(cuda_dev),
                   rand_feat=torch.from_numpy(g['rand_feat']).to(cuda_dev),
                   rand_feat_color=torch.from_numpy(g['rand_feat_color']).to(cuda_dev))
        o2 = model(inp)
    assert torch.equal(o2['rgb'], out['rgb']) and torch.equal(o2['depth'], out['depth'])


@pytest.mark.gpu
@pytest.mark.parametrize('N', [1, 777, 200000])
def test_knn_index_device_build_equals_stable_argsort(cuda_dev, N):
    """xrd_pointslam_knn_build (histogram / scan / scatter / per-bucket sort on the device) ==
    the torch construction it replaces (stable argsort of the bucket keys), bit for bit."""
    from xrdslam_b200.neural_point_cloud import NeuralPointCloud
    npc = NeuralPointCloud(device=cuda_dev)
    g = torch.Generator().manual_seed(N)
    pos = (torch.rand(N, 3, generator=g) - 0.5) * torch.tensor([6.0, 6.0, 3.0])
    pos[: N // 3] = pos[: N // 3].round(decimals=1)  # crowded cells
    npc.set_cloud(pos, torch.zeros(N, 32))
    npc.rebuild_index()
    ref = npc.rebuild_index_torch()
    torch.cuda.synchronize()
    for k in ('cell_start', 'cell_end'):
        assert torch.equal(npc._index[k], ref[k]), k
    assert torch.equal(npc._index['sorted_ids'][:N], ref['sorted_ids'])
