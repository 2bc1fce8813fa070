"""Co-SLAM with a separate colour hash grid (oneGrid=False, ColorSDFNet): the fused step
(k_fused_c), the mesher queries (k_query_c), the graph sessions and a short run, against the
two-grid oracle (oracle/coslam_color_grid.py) and the generic autograd path."""
import ctypes as C
import random

import numpy as np
import pytest
import torch

from helpers import BOUND, make_rays, max_abs, rel_err

pytestmark = pytest.mark.gpu

TOL_OUT = 2e-5     # abs
TOL_LOSS = 2e-5    # rel
TOL_GRAD = 2e-4    # rel l2
# precision 1 (TF32 backward) gradients, precision 2 (TF32 everywhere) outputs and losses
TOL_GRAD_TF32 = 5e-3
TOL_OUT_TF32, TOL_LOSS_TF32 = 5e-2, 3e-2


def color_pair(device, table_amp=0.3, seed=1, **cfg):
    """(two-grid oracle on CPU, CUDA model with oneGrid=False on device), same parameters."""
    from oracle.coslam_color_grid import CoslamColorGridOracle
    from xrdslam_b200.camera import Camera
    from xrdslam_b200.joint_encoding import JointEncodingConfig
    ora = CoslamColorGridOracle(BOUND)
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for enc in (ora.embed_fn, ora.embed_fn_color):
            enc.params.copy_((torch.rand(enc.params.shape, generator=g) * 2 - 1) * table_amp)
        for lin in (ora.sdf0, ora.sdf1, ora.col0, ora.col1):
            lin.weight.copy_(torch.randn(lin.weight.shape, generator=g) *
                             (1.0 / np.sqrt(lin.weight.shape[1])))
    model = JointEncodingConfig(oneGrid=False, **cfg).setup(
        camera=Camera(320., 320., 319.5, 239.5, 640, 480), bounding_box=BOUND)
    with torch.no_grad():
        model.embed_fn.params.copy_(ora.embed_fn.params)
        model.embed_fn_color.params.copy_(ora.embed_fn_color.params)
        model.decoder.sdf_net.model[0].weight.copy_(ora.sdf0.weight)
        model.decoder.sdf_net.model[2].weight.copy_(ora.sdf1.weight)
        model.decoder.color_net.model[0].weight.copy_(ora.col0.weight)
        model.decoder.color_net.model[2].weight.copy_(ora.col1.weight)
    model.to(device)
    return ora, model


def _pairs(model, ora):
    d = model.decoder
    return [(model.embed_fn.params, ora.embed_fn.params),
            (model.embed_fn_color.params, ora.embed_fn_color.params),
            (d.sdf_net.model[0].weight, ora.sdf0.weight), (d.sdf_net.model[2].weight, ora.sdf1.weight),
            (d.color_net.model[0].weight, ora.col0.weight), (d.color_net.model[2].weight, ora.col1.weight)]


def test_color_grid_hash_indices_bit_exact(cuda_dev):
    from oracle.tcnn_restated import hashgrid_indices
    from xrdslam_b200 import _cabi
    ora, model = color_pair(cuda_dev)
    g = torch.Generator().manual_seed(5)
    x = torch.rand(20000, 3, generator=g) * 3 - 1  # in and outside [0,1]
    idx_o, _ = hashgrid_indices(x, ora.embed_fn_color.table)
    feat = torch.empty(x.shape[0], 32, device=cuda_dev)
    idx = torch.empty(x.shape[0], 16, 8, dtype=torch.int32, device=cuda_dev)
    grid = model._grid_struct(model.embed_fn_color.params.detach(), model.embed_fn_color)
    _cabi.check('xrd_hashgrid_encode', _cabi.lib().xrd_hashgrid_encode(
        C.byref(grid), x.to(cuda_dev).data_ptr(), x.shape[0], feat.data_ptr(), idx.data_ptr(), None))
    torch.cuda.synchronize()
    assert torch.equal(idx.cpu().to(torch.int64) & 0xFFFFFFFF, idx_o)
    with torch.no_grad():
        assert max_abs(feat, ora.embed_fn_color(x)) < 1e-6


@pytest.mark.parametrize('precision', [0, 1, 2])
@pytest.mark.parametrize('R', [1, 5, 257, 1024, 4096])
def test_step_parity(cuda_dev, R, precision):
    ora, model = color_pair(cuda_dev, precision=precision)
    rays_o, rays_d, ts, td, noise = make_rays(R, seed=R)
    rays_o.requires_grad_(True)
    rays_d.requires_grad_(True)
    out_o, ld_o, tot_o = ora.step(rays_o, rays_d, ts, td, noise, False, True)
    tot_o.backward()
    ro = rays_o.detach().to(cuda_dev).requires_grad_(True)
    rd = rays_d.detach().to(cuda_dev).requires_grad_(True)
    inp = dict(rays_o=ro, rays_d=rd, target_s=ts.to(cuda_dev), target_d=td.to(cuda_dev),
               first=True, noise=noise.to(cuda_dev))
    out = model(inp)
    ld = model.get_loss_dict(out, inp, False, 0)
    sum(ld.values()).backward()
    torch.cuda.synchronize()
    assert torch.equal(out['z_vals'].cpu(), out_o['z_vals'])
    t_out, t_loss = (TOL_OUT_TF32, TOL_LOSS_TF32) if precision == 2 else (TOL_OUT, TOL_LOSS)
    if precision == 2:
        # TF32 sdf values can move a ray's first sign change (and with it the sample mask), so
        # a few rays of a large batch differ by more: 99 % of them stay within the tolerance
        for k in ('rgb', 'depth'):
            err = (out[k].detach().cpu().double() - out_o[k].detach().double()).abs()
            err = err.reshape(R, -1).amax(-1)
            assert float((err < t_out).double().mean()) >= 0.99, k
    else:
        for k in ('rgb', 'depth', 'acc_map', 'depth_var'):
            assert max_abs(out[k], out_o[k]) < t_out, k
    for k in ld_o:
        a, b = float(ld[k].detach()), float(ld_o[k].detach())
        assert abs(a - b) <= t_loss * max(abs(b), 1e-6), (k, a, b)
    assert model.embed_fn_color.params.grad.abs().max() > 0
    if precision == 2:
        for m, o in _pairs(model, ora)[:2]:
            ga, gb = m.grad.cpu().double(), o.grad.double()
            assert float((ga * gb).sum() / (ga.norm() * gb.norm())) > 0.995
        return
    tol = TOL_GRAD if precision == 0 else TOL_GRAD_TF32
    for i, (m, o) in enumerate(_pairs(model, ora)):
        assert rel_err(m.grad, o.grad) < tol, i
    assert rel_err(ro.grad, rays_o.grad) < tol
    assert rel_err(rd.grad, rays_d.grad) < tol


@pytest.mark.parametrize('R', [257, 1024])
def test_step_in_kernel_noise_matches_oracle(cuda_dev, R):
    """No explicit noise: the kernel draws the jitter; the oracle replays the z samples it chose
    (z_vals are a function of the noise only), so every other output is compared as above."""
    ora, model = color_pair(cuda_dev)
    rays_o, rays_d, ts, td, _ = make_rays(R, seed=R + 1)
    inp = dict(rays_o=rays_o.to(cuda_dev), rays_d=rays_d.to(cuda_dev), target_s=ts.to(cuda_dev),
               target_d=td.to(cuda_dev), first=True)
    out = model(inp)
    ld = model.get_loss_dict(out, inp, False, 0)
    sum(ld.values()).backward()
    z = out['z_vals'].detach().cpu()
    ora.sample_z = lambda n_rays, target_d, noise: z  # the kernel's samples
    out_o, ld_o, tot_o = ora.step(rays_o, rays_d, ts, td, None, False, True)
    tot_o.backward()
    for k in ('rgb', 'depth'):
        assert max_abs(out[k], out_o[k]) < TOL_OUT, k
    for k in ld_o:
        a, b = float(ld[k].detach()), float(ld_o[k].detach())
        assert abs(a - b) <= TOL_LOSS * max(abs(b), 1e-6), (k, a, b)
    for i, (m, o) in enumerate(_pairs(model, ora)):
        assert rel_err(m.grad, o.grad) < TOL_GRAD, i


def test_pose_only_pass(cuda_dev):
    """Tracking: map gradients off, the colour grid still adds to d rays."""
    ora, model = color_pair(cuda_dev)
    rays_o, rays_d, ts, td, noise = make_rays(1024, seed=9)
    rays_o.requires_grad_(True)
    rays_d.requires_grad_(True)
    _, _, tot_o = ora.step(rays_o, rays_d, ts, td, noise, False, True)
    tot_o.backward()
    model.freeze_map_grads = True
    ro = rays_o.detach().to(cuda_dev).requires_grad_(True)
    rd = rays_d.detach().to(cuda_dev).requires_grad_(True)
    inp = dict(rays_o=ro, rays_d=rd, target_s=ts.to(cuda_dev), target_d=td.to(cuda_dev),
               first=False, noise=noise.to(cuda_dev))
    sum(model.get_loss_dict(model(inp), inp, False, 0).values()).backward()
    torch.cuda.synchronize()
    assert rel_err(ro.grad, rays_o.grad) < TOL_GRAD
    assert rel_err(rd.grad, rays_d.grad) < TOL_GRAD
    assert model.embed_fn_color.params.grad is None or not model.embed_fn_color.params.grad.any()


def test_render_forward_only(cuda_dev):
    ora, model = color_pair(cuda_dev)
    rays_o, rays_d, ts, td, noise = make_rays(700, seed=4)
    with torch.no_grad():
        out_o = ora.render_rays(rays_o, rays_d, td, noise)
        out = model(dict(rays_o=rays_o.to(cuda_dev), rays_d=rays_d.to(cuda_dev),
                         target_d=td.to(cuda_dev), noise=noise.to(cuda_dev)))
    for k in ('rgb', 'depth', 'acc_map', 'depth_var'):
        assert max_abs(out[k], out_o[k]) < TOL_OUT, k
    assert max_abs(out['raw'], out_o['raw']) < 5e-5


def test_kernel_choice(cuda_dev):
    """Automatic choice runs a colour-grid gradient pass on the tile kernel (bit-equal outputs to
    rays_per_tile = -1 at a batch the one-grid path sends to the grouped kernel); -2 refuses."""
    from xrdslam_b200 import _cabi
    outs = []
    rays_o, rays_d, ts, td, noise = make_rays(4096, seed=2)
    for rpt in (0, -1):
        _, model = color_pair(cuda_dev, rays_per_tile=rpt)
        w = model._weights()
        o, _ = model._launch(rays_o.to(cuda_dev), rays_d.to(cuda_dev), model.embed_fn.params, *w,
                             ts.to(cuda_dev), td.to(cuda_dev), noise.to(cuda_dev), with_grads=True)
        outs.append(o)
    for k in ('rgb', 'depth', 'raw', 'losses'):
        assert torch.equal(outs[0][k], outs[1][k]), k
    _, model = color_pair(cuda_dev, rays_per_tile=-2)
    w = model._weights()
    with pytest.raises(_cabi.XrdError) as e:
        model._launch(rays_o.to(cuda_dev), rays_d.to(cuda_dev), model.embed_fn.params, *w,
                      ts.to(cuda_dev), td.to(cuda_dev), noise.to(cuda_dev), with_grads=True)
    assert 'XRD_E_SHAPE' in str(e.value)


def test_queries_match_oracle(cuda_dev):
    ora, model = color_pair(cuda_dev)
    g = torch.Generator().manual_seed(8)
    x = torch.rand(5000, 3, generator=g)
    with torch.no_grad():
        raw_o = ora.query_color_sdf(x)
        raw = model.query_color_sdf(x.to(cuda_dev))
        assert max_abs(raw, raw_o) < 1e-5
        pts = torch.from_numpy(BOUND[:, 0] + x.double().numpy() * (BOUND[:, 1] - BOUND[:, 0])).float()
        raw_w = model.run_network(pts.to(cuda_dev))
        assert max_abs(raw_w, ora.query_color_sdf(ora.normalise(pts.double()))) < 1e-4
        # query_sdf(embed=True) is the SDF grid's encoding
        assert max_abs(model.query_sdf(x.to(cuda_dev), embed=True), ora.embed_fn(x)) < 1e-6


def _build_algorithm(dev, seed):
    """bench.build_algorithm with oneGrid=False."""
    import bench
    from xrdslam_b200.coslam import CoSLAMConfig
    from xrdslam_b200.frame import Frame
    from xrdslam_b200.synthetic import make_sequence
    random.seed(seed)
    np.random.seed(seed)
    torch.manual_seed(seed)
    cam, poses, frames = make_sequence(bench.N_KEYFRAMES + 1)
    cfg = CoSLAMConfig()
    cfg.model.precision = 1
    cfg.model.oneGrid = False
    algo = cfg.setup(camera=cam, device=dev)
    kfs = []
    for k in range(bench.N_KEYFRAMES):
        f = Frame(k, frames[k][0], frames[k][1], init_pose=poses[k], separate_LR=True,
                  rot_rep='axis_angle')
        algo.add_keyframe(f)
        kfs.append(f)
    cur = Frame(bench.N_KEYFRAMES, frames[-1][0], frames[-1][1], init_pose=poses[-1],
                separate_LR=True, rot_rep='axis_angle')
    algo.set_initialized()
    return algo, kfs, cur


def _map(dev, graph, n_iters, seed=11):
    random.seed(seed)
    algo, kfs, cur = _build_algorithm(dev, seed)
    algo.config.graph_mapping = graph
    algo.config.min_sample_pixels = 256
    frames = kfs + [cur]
    torch.manual_seed(seed)
    losses = []
    if graph:
        algo.setup_optimizers(n_iters, frames, True)
        sess = algo.mapping_session(frames)
        assert 'embed_fn_color' in sess.group_names
        sess.begin(frames)
        for i in range(n_iters):
            losses.append(float(sess.step(i, frames)))
        sess.end(frames)
    else:
        orig = algo.get_loss

        def wrapped(*a, **k):
            loss = orig(*a, **k)
            losses.append(float(loss.detach()))
            return loss
        algo.get_loss = wrapped
        algo.optimize_update(n_iters, frames, True)
    return algo, frames, losses


def test_graph_mapping_matches_generic_path(cuda_dev):
    a_g, f_g, l_g = _map(cuda_dev, True, 7)
    a_e, f_e, l_e = _map(cuda_dev, False, 7)
    assert len(l_g) == len(l_e) == 7
    for x, y in zip(l_g, l_e):
        assert abs(x - y) <= 2e-3 * abs(y), (l_g, l_e)
    assert l_g[-1] < l_g[0]
    for p, q in zip(a_g.model.decoder.parameters(), a_e.model.decoder.parameters()):
        assert (p - q).abs().max() <= 2e-3 * q.abs().max()
    # Adam with eps = 1e-15 steps every entry by about lr whatever its gradient's size, so entries
    # whose gradient is near zero amplify the atomic summation order: a looser bound than above
    cg, ce = a_g.model.embed_fn_color.params, a_e.model.embed_fn_color.params
    assert rel_err(cg, ce) < 1e-2
    assert not torch.equal(cg.detach().cpu(), _build_algorithm(cuda_dev, 11)[0].model.embed_fn_color.params.detach().cpu())
    for fg, fe in zip(f_g, f_e):
        assert (fg.pose.data_t - fe.pose.data_t).abs().max() < 2e-5
        assert (fg.pose.data_r - fe.pose.data_r).abs().max() < 2e-5


def test_tracking_graph_matches_generic_iteration(cuda_dev):
    from xrdslam_b200.common import sample_window
    from xrdslam_b200.coslam_graph import TrackingGraphSession
    from xrdslam_b200.opt_pose import pose_matrices
    algo, kfs, cur = _build_algorithm(cuda_dev, 3)
    algo.config.graph_mapping = False
    cam = algo.camera
    He, We, n = algo.config.tracking_Hedge, algo.config.tracking_Wedge, algo.config.tracking_sample
    g = torch.Generator().manual_seed(0)
    idx = torch.randint((cam.height - 2 * He) * (cam.width - 2 * We), (n,), generator=g).to(cuda_dev)
    sess = TrackingGraphSession(algo, external_indices=True)
    r0, t0 = cur.pose.data_r.detach().clone(), cur.pose.data_t.detach().clone()
    sess.begin(cur)
    sess.idx.copy_(idx)
    c0 = algo.model._step_count
    loss_g = float(sess.step())
    d_rot_g, d_trans_g = sess.d_rot.cpu().reshape(3), sess.d_trans.cpu().reshape(3)
    sess.end(cur)
    with torch.no_grad():
        cur.pose.data_r.copy_(r0)
        cur.pose.data_t.copy_(t0)
    algo.model._step_count = c0
    algo.model.freeze_map_grads = True
    opt = algo.setup_optimizers(1, [cur], is_mapping=False)
    opt.zero_grad_all()
    ro, rd, d, c = sample_window(cam, [algo._frame_tensor(cur, 'depth')], [algo._frame_tensor(cur, 'rgb')],
                                 pose_matrices([cur.pose]).to(cuda_dev), n, He, We, indices=idx)
    inp = dict(rays_o=ro, rays_d=rd, target_s=c, target_d=d, first=False)
    loss = sum(algo.model.get_loss_dict(algo.model(inp), inp, False, 0).values())
    loss.backward()
    assert abs(loss_g - float(loss.detach())) <= 1e-5 * abs(float(loss.detach()))
    assert (d_rot_g - cur.pose.data_r.grad).abs().max() <= 1e-4 * cur.pose.data_r.grad.abs().max()
    assert (d_trans_g - cur.pose.data_t.grad).abs().max() <= 1e-4 * cur.pose.data_t.grad.abs().max()


def test_run_and_eval_color_grid(cuda_dev, tmp_path):
    """A short synthetic Replica run with model.oneGrid=False through get_mesh (vertex colours
    from the colour grid) and ds-eval."""
    import math
    import os
    import warnings

    from test_pipeline_gpu import HEIGHT, N_FRAMES, REDUCED, TURN, WIDTH
    from xrdslam_b200.eval import EvalMatrics
    from xrdslam_b200.io_formats import write_ply
    from xrdslam_b200.pipeline import XRDSLAM, make_config
    from xrdslam_b200.synthetic import room_mesh, write_replica
    torch.manual_seed(0)
    np.random.seed(0)
    folder = tmp_path / 'replica'
    write_replica(str(folder), N_FRAMES, width=WIDTH, height=HEIGHT, turn=TURN)
    v, f = room_mesh()
    gt = str(tmp_path / 'room.ply')
    write_ply(gt, v, f)
    out = tmp_path / 'out'
    cfg = make_config('co-slam', data=str(folder), out_dir=str(out), device=str(cuda_dev),
                      **REDUCED['co-slam'], **{'model.oneGrid': False})
    assert cfg.algorithm.model.oneGrid is False
    with warnings.catch_warnings():
        warnings.simplefilter('ignore', UserWarning)
        res = XRDSLAM(cfg).run()
    assert res['n_frames'] == N_FRAMES
    for name in ('eval.tar', 'final_mesh.ply', 'final_mesh_rec.ply'):
        assert os.path.exists(out / name), name
    m = EvalMatrics(output_dir=out, gt_mesh=gt, device=str(cuda_dev)).main()
    assert math.isfinite(float(m['accuracy'])) and math.isfinite(float(m['completion']))


def test_render_without_depth(cuda_dev):
    """target_d=None -> 256 uniform samples: one ray of 256 points per tile, on the compact
    forward-only record."""
    ora, model = color_pair(cuda_dev)
    rays_o, rays_d, _, _, _ = make_rays(300, seed=6)
    noise = torch.rand(300, 256, generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        out_o = ora.render_rays(rays_o, rays_d, None, noise)
        out = model(dict(rays_o=rays_o.to(cuda_dev), rays_d=rays_d.to(cuda_dev),
                         noise=noise.to(cuda_dev)))
    assert torch.equal(out['z_vals'].cpu(), out_o['z_vals'])
    for k in ('rgb', 'depth', 'acc_map'):
        assert max_abs(out[k], out_o[k]) < TOL_OUT, k
    assert max_abs(out['raw'], out_o['raw']) < 5e-5


def test_step_matches_reference_golden(cuda_dev):
    """The fused step against what the reference's own JointEncoding(oneGrid=False) returned
    (tests/golden/make_golden_coslam_color_grid.py): outputs, losses, both tables, the four
    weights and the rays."""
    from test_coslam_color_grid_cpu import GOLDEN, LOSS_KEYS, WEIGHTS, color_grid_case
    g = np.load(GOLDEN)
    ora, (rays_o, rays_d, ts, td, noise) = color_grid_case()
    _, model = color_pair(cuda_dev)
    sd = dict(model.named_parameters())
    with torch.no_grad():
        model.embed_fn.params.copy_(ora.embed_fn.params)
        model.embed_fn_color.params.copy_(ora.embed_fn_color.params)
        for name, key in WEIGHTS:
            sd[key].copy_(getattr(ora, name).weight)
    ro = rays_o.to(cuda_dev).requires_grad_(True)
    rd = rays_d.to(cuda_dev).requires_grad_(True)
    inp = dict(rays_o=ro, rays_d=rd, target_s=ts.to(cuda_dev), target_d=td.to(cuda_dev),
               first=True, noise=noise.to(cuda_dev))
    out = model(inp)
    ld = model.get_loss_dict(out, inp, False, 0)
    sum(ld.values()).backward()
    torch.cuda.synchronize()
    assert np.array_equal(out['z_vals'].cpu().numpy(), g['z_vals'])
    for k in ('rgb', 'depth', 'acc_map', 'depth_var'):
        assert max_abs(out[k], g[k]) < TOL_OUT, k
    for i, k in enumerate(LOSS_KEYS):
        a, b = float(ld[k].detach()), float(g['losses'][i])
        assert abs(a - b) <= TOL_LOSS * max(abs(b), 1e-6), (k, a, b)
    for key, t in (('d_table', model.embed_fn.params), ('d_table_color', model.embed_fn_color.params)):
        dense = torch.zeros(t.numel() // 2, 2, dtype=torch.float64)
        dense[torch.from_numpy(g[key + '.idx']).long()] = torch.from_numpy(g[key + '.val']).double()
        assert rel_err(t.grad, dense) < TOL_GRAD, key
    for name, key in WEIGHTS:
        assert rel_err(sd[key].grad, g['d_' + name]) < TOL_GRAD, key
    assert rel_err(ro.grad, g['d_rays_o']) < TOL_GRAD
    assert rel_err(rd.grad, g['d_rays_d']) < TOL_GRAD


@pytest.mark.parametrize('pass_', ['mapping', 'pose-only'])
def test_step_vs_float64_per_entry(cuda_dev, pass_):
    """The step against the two-grid oracle evaluated in float64 on the kernel's discrete inputs
    (z samples, fp32 hash indices and cell fractions): every entry of both tables, every element
    of w_col0 [32, 95] and every ray.  An entry the float64 step leaves at zero gets exactly
    zero, and every other one is within 2e-3 of its own magnitude plus 1e-4 of its level's
    largest: a scatter to a wrong entry, or a lost one, fails here even where the relative L2
    over the table would not see it.  Rays whose first sdf sign change the fp32 and float64 steps
    put at different samples are left out, with the entries their points touch."""
    from oracle.tcnn_restated import hashgrid_indices
    ora, model = color_pair(cuda_dev)
    R = 257
    rays_o, rays_d, ts, td, noise = make_rays(R, seed=31)
    ro = rays_o.to(cuda_dev).requires_grad_(True)
    rd = rays_d.to(cuda_dev).requires_grad_(True)
    inp = dict(rays_o=ro, rays_d=rd, target_s=ts.to(cuda_dev), target_d=td.to(cuda_dev),
               first=True, noise=noise.to(cuda_dev))
    model.freeze_map_grads = pass_ == 'pose-only'
    out = model(inp)
    sum(model.get_loss_dict(out, inp, False, 0).values()).backward()
    torch.cuda.synchronize()
    z = out['z_vals'].detach().cpu()
    o64 = ora.double()
    o64.sample_z = lambda n_rays, target_d, noise: z.double()
    r64o, r64d = rays_o.double().requires_grad_(True), rays_d.double().requires_grad_(True)
    out64, _, tot64 = o64.step(r64o, r64d, ts.double(), td.double(), None, False, True)
    tot64.backward()

    def first_change(sdf):
        return torch.argmax(((sdf[:, 1:] * sdf[:, :-1]) < 0).int(), dim=1)
    flip = first_change(out['raw'][..., 3].detach().cpu()) != first_change(out64['raw'][..., 3].detach())
    keep_rays = ~flip
    assert int(flip.sum()) <= R // 50, int(flip.sum())
    pts = (rays_o[:, None, :] + rays_d[:, None, :] * z[..., None])[flip].reshape(-1, 3)
    x32 = ((pts.double() - o64.bounding_box[:, 0]) / (o64.bounding_box[:, 1] - o64.bounding_box[:, 0])).float()

    def close(g, r, scale):
        return (g - r).abs() <= 2e-3 * r.abs() + 1e-4 * scale

    for d, r in ((ro.grad.cpu().double(), r64o.grad), (rd.grad.cpu().double(), r64d.grad)):
        assert bool(close(d, r, r.abs().max())[keep_rays].all())
    if pass_ == 'pose-only':
        assert model.embed_fn_color.params.grad is None or not model.embed_fn_color.params.grad.any()
        return
    gw, rw = model.decoder.color_net.model[0].weight.grad.cpu().double(), o64.col0.weight.grad
    assert gw.shape == (32, 95)
    if not bool(flip.any()):
        assert bool(close(gw, rw, rw.abs().max()).all())
    for enc_m, enc_o in ((model.embed_fn, o64.embed_fn), (model.embed_fn_color, o64.embed_fn_color)):
        g = enc_m.params.grad.cpu().double().reshape(-1, 2)
        r = enc_o.params.grad.reshape(-1, 2)
        skip = torch.zeros(g.shape[0], dtype=torch.bool)
        if bool(flip.any()):
            idx, _ = hashgrid_indices(x32, enc_o.table)
            skip[idx.reshape(-1)] = True
        lay = enc_o.table
        for o, n in zip(lay['offset'], lay['size']):
            a, b = int(o), int(o) + int(n)
            gl, rl, kl = g[a:b], r[a:b], ~skip[a:b]
            assert bool((gl[kl][rl[kl] == 0] == 0).all())
            assert bool(close(gl, rl, rl.abs().max())[kl].all()), (a, b)
