"""Co-SLAM importance sampling (training_n_importance > 0): the device sample_pdf
(xrd_coslam_importance), the coarse + fine fused step through both kernels, the pose-only pass,
the colour grid, forward rendering, the graph sessions and a short run, against the importance
oracle (oracle/coslam_importance.py) and the generic autograd path."""
import random

import numpy as np
import pytest
import torch

from helpers import coslam_pair, make_rays, max_abs, rel_err

pytestmark = pytest.mark.gpu

TOL_OUT = 2e-5     # abs
TOL_LOSS = 2e-5    # rel
TOL_GRAD = 2e-4    # rel l2
TOL_GRAD_TF32 = 5e-3  # precision 1: TF32 backward
OUTS = ('rgb', 'depth', 'acc_map', 'depth_var', 'rgb0', 'depth0', 'acc0', 'depth_var0')


def _weights(model, ora):
    d = model.decoder
    return [(model.embed_fn.params, ora.embed_fn.params),
            (d.sdf_net.model[0].weight, ora.sdf0.weight), (d.sdf_net.model[2].weight, ora.sdf1.weight),
            (d.color_net.model[0].weight, ora.col0.weight), (d.color_net.model[2].weight, ora.col1.weight)]


def _importance(model, dev, z, raw, td, u=None, seed=0, counts=None):
    """xrd_coslam_importance on a coarse pass given on the host -> its buffers."""
    import ctypes as C
    from xrdslam_b200 import _cabi
    R, S = z.shape
    b, q = model._importance_struct(R, S, dev, z.to(dev), raw.to(dev), td.reshape(-1).to(dev),
                                    None if u is None else u.to(dev), seed=seed, counts=counts)
    _cabi.launch_on(dev, 'xrd_coslam_importance', C.byref(q))
    torch.cuda.synchronize()
    return b


@pytest.mark.parametrize('det', [False, True])  # u given [R,N]; the det linspace table
def test_sampler_matches_oracle(cuda_dev, det):
    """The device sample_pdf on the coarse pass of the oracle (same raw, same z_vals, same u).
    The two cdfs agree to a few float ulps (the kernel's sigmoid and sum orders are not torch's),
    so a sample agrees to 1e-3 of its bin width unless that ulp difference is amplified: u within
    float rounding of a cdf value (the searchsorted index may differ by one) or a bin whose cdf
    step (the denominator) is small.  Those are counted and bounded.  The merged z_vals are
    sorted, the fine pass's counts and z_std follow from them."""
    from oracle import coslam_importance as CI
    N, R = 16, 4096
    ora, model = coslam_pair(cuda_dev, training_n_importance=N, training_perturb=0 if det else 1)
    ora.cfg.perturb = 0 if det else 1
    rays_o, rays_d, ts, td, noise = make_rays(R, seed=3)
    if det:
        u = CI.det_u(N).expand(R, N)
    else:
        u = torch.rand(R, N, generator=torch.Generator().manual_seed(4))
    with torch.no_grad():
        co = ora.render_rays(rays_o, rays_d, td, noise)
    z, raw = co['z_vals'], co['raw']
    mid = .5 * (z[..., 1:] + z[..., :-1])
    zs_o, inds, cdf = CI.sample_pdf(mid, co['weights'][..., 1:-1], u)
    counts = torch.zeros(4, dtype=torch.int32, device=cuda_dev)
    # det: no u given, the kernel reads the model's linspace table
    b = _importance(model, cuda_dev, z, raw, td, None if det else u, counts=counts)
    zs = b['z_samples'].cpu()
    below = (inds - 1).clamp(min=0)
    above = inds.clamp(max=cdf.shape[-1] - 1)
    binw = (mid.gather(1, above) - mid.gather(1, below)).clamp(min=1e-12)
    off = (zs - zs_o).abs() / binw
    near_cdf = ((u[..., None] - cdf[:, None, :]).abs() < 1e-6).any(-1)
    den = cdf.gather(1, above) - cdf.gather(1, below)
    den = torch.where(den < 1e-5, torch.ones_like(den), den)
    ulp_amplified = off <= 8 * 1.2e-7 / den  # eight ulps of a cdf value near 1, over the step
    bad = off > 1e-3
    print(f'sampler: {int(bad.sum())} of {zs.numel()} samples off by > 1e-3 bin widths '
          f'({int((bad & near_cdf).sum())} with u within 1e-6 of a cdf value); '
          f'median offset {float(off.median()):.3g}, max of the others {float(off[~bad].max()):.3g}')
    assert float(bad.double().mean()) < 1e-3
    assert bool(torch.all(near_cdf[bad] | ulp_amplified[bad]))
    assert float(off.median()) < 1e-5
    zf = b['z_vals'].cpu()
    assert torch.all(zf[:, 1:] >= zf[:, :-1])
    assert torch.equal(zf, torch.sort(torch.cat([z, zs], -1), -1)[0])
    # the fine pass's loss normalisers over the merged samples
    tr = ora.cfg.trunc
    front = zf < td - tr
    back = zf > td + tr
    n_sdf = int(((~front) & (~back) & (td > 0)).sum())
    valid = int(((td > 0) & (td < ora.cfg.depth_trunc)).sum())
    assert counts.cpu().tolist()[:3] == [int(front.sum()), n_sdf, valid]
    assert max_abs(b['z_std'], zs.double().std(-1, unbiased=False)) < 2e-6
    if det:
        assert torch.all(zs[:, 1:] >= zs[:, :-1])


def test_sampler_philox_draws(cuda_dev):
    """No u given and training_perturb > 0: Philox uniforms from the seed.  The same seed gives
    the same samples, another seed other samples, and the uniforms read back through the cdf
    (u = cdf[j] + t (cdf[j+1] - cdf[j]) of the bin a sample lies in) are uniform on [0, 1)."""
    from oracle import coslam_importance as CI
    N, R = 16, 4096
    ora, model = coslam_pair(cuda_dev, training_n_importance=N)
    rays_o, rays_d, ts, td, noise = make_rays(R, seed=3)
    with torch.no_grad():
        co = ora.render_rays(rays_o, rays_d, td, noise)
    z, raw = co['z_vals'], co['raw']
    zs = [_importance(model, cuda_dev, z, raw, td, seed=s)['z_samples'].cpu() for s in (7, 7, 8)]
    assert torch.equal(zs[0], zs[1])
    assert float((zs[0] != zs[2]).double().mean()) > 0.99
    mid = .5 * (z[..., 1:] + z[..., :-1])
    _, _, cdf = CI.sample_pdf(mid, co['weights'][..., 1:-1], torch.zeros(R, 1))
    for x in (zs[0], zs[2]):
        j = (torch.searchsorted(mid, x, right=True) - 1).clamp(0, mid.shape[1] - 2)
        m0, m1 = mid.gather(1, j), mid.gather(1, j + 1)
        c0, c1 = cdf.gather(1, j).double(), cdf.gather(1, j + 1).double()
        u = c0 + ((x - m0) / (m1 - m0)).double() * (c1 - c0)
        assert float(u.min()) >= -1e-5 and float(u.max()) <= 1 + 1e-5
        assert abs(float(u.mean()) - 0.5) < 0.01
        assert abs(float(u.std()) - 12 ** -0.5) < 0.01
        hist = torch.histc(u.float().clamp(0, 1 - 1e-7), bins=10, min=0, max=1) / u.numel()
        assert float((hist - 0.1).abs().max()) < 0.01, hist


def _step(cuda_dev, model, ora, R, N, seed=0, fused=True):
    """(GPU outputs, losses, gradients) and the oracle's on the GPU's fine z_vals."""
    from oracle import coslam_importance as CI
    rays_o, rays_d, ts, td, noise = make_rays(R, seed=R + seed)
    u = torch.rand(R, N, generator=torch.Generator().manual_seed(R))
    rays_o.requires_grad_(True)
    rays_d.requires_grad_(True)
    ro = rays_o.detach().to(cuda_dev).requires_grad_(True)
    rd = rays_d.detach().to(cuda_dev).requires_grad_(True)
    inp = dict(rays_o=ro, rays_d=rd, target_s=ts.to(cuda_dev), target_d=td.to(cuda_dev),
               first=True, noise=noise.to(cuda_dev), importance_u=u.to(cuda_dev))
    out = model(inp)
    ld = model.get_loss_dict(out, inp, False, 0)
    sum(ld.values()).backward()
    torch.cuda.synchronize()
    assert out['z_vals'].shape == (R, 43 + N)
    out_o, ld_o, tot_o = CI.step(ora, rays_o, rays_d, ts, td, noise, u,
                                 z_fine=out['z_vals'].detach().cpu())
    tot_o.backward()
    return out, ld, (ro, rd), out_o, ld_o, (rays_o, rays_d)


def _check(model, ora, out, ld, rays, out_o, ld_o, rays_oo, tol_grad=TOL_GRAD):
    for k in OUTS:
        assert max_abs(out[k], out_o[k]) < TOL_OUT, k
    for k in ld_o:
        a, b = float(ld[k].detach()), float(ld_o[k].detach())
        assert abs(a - b) <= TOL_LOSS * max(abs(b), 1e-6), (k, a, b)
    for i, (m, o) in enumerate(_weights(model, ora)):
        assert rel_err(m.grad, o.grad) < tol_grad, i
    for a, b in zip(rays, rays_oo):
        assert rel_err(a.grad, b.grad) < tol_grad


@pytest.mark.parametrize('N', [16, 53])  # 53: S0 + N = 96, the grouped kernel's limit
@pytest.mark.parametrize('kernel', [-1, -2, 0])  # tile, grouped, automatic
@pytest.mark.parametrize('precision', [0, 1])
def test_step_parity(cuda_dev, N, kernel, precision):
    ora, model = coslam_pair(cuda_dev, training_n_importance=N, rays_per_tile=kernel,
                             precision=precision)
    R = 1024
    res = _step(cuda_dev, model, ora, R, N)
    _check(model, ora, *res[:3], *res[3:], tol_grad=TOL_GRAD if precision == 0 else TOL_GRAD_TF32)


def test_pose_only_pass(cuda_dev):
    """Tracking: only the ray gradients, summed over both passes."""
    from oracle import coslam_importance as CI
    N, R = 16, 1024
    ora, model = coslam_pair(cuda_dev, training_n_importance=N)
    model.freeze_map_grads = True
    rays_o, rays_d, ts, td, noise = make_rays(R, seed=8)
    u = torch.rand(R, N, generator=torch.Generator().manual_seed(8))
    ro = rays_o.to(cuda_dev).requires_grad_(True)
    rd = rays_d.to(cuda_dev).requires_grad_(True)
    inp = dict(rays_o=ro, rays_d=rd, target_s=ts.to(cuda_dev), target_d=td.to(cuda_dev),
               first=False, noise=noise.to(cuda_dev), importance_u=u.to(cuda_dev))
    for p in model.parameters():
        p.requires_grad_(False)
    out = model(inp)
    sum(model.get_loss_dict(out, inp, False, 0).values()).backward()
    rays_o.requires_grad_(True)
    rays_d.requires_grad_(True)
    _, _, tot = CI.step(ora, rays_o, rays_d, ts, td, noise, u, z_fine=out['z_vals'].cpu())
    tot.backward()
    assert rel_err(ro.grad, rays_o.grad) < TOL_GRAD
    assert rel_err(rd.grad, rays_d.grad) < TOL_GRAD


def test_color_grid_with_importance(cuda_dev):
    from test_coslam_color_grid_gpu import _pairs, color_pair
    N, R = 16, 1024
    ora, model = color_pair(cuda_dev, training_n_importance=N)
    res = _step(cuda_dev, model, ora, R, N)
    out, ld, rays, out_o, ld_o, rays_oo = res
    for k in OUTS:
        assert max_abs(out[k], out_o[k]) < TOL_OUT, k
    for k in ld_o:
        a, b = float(ld[k].detach()), float(ld_o[k].detach())
        assert abs(a - b) <= TOL_LOSS * max(abs(b), 1e-6), (k, a, b)
    for i, (m, o) in enumerate(_pairs(model, ora)):
        assert rel_err(m.grad, o.grad) < TOL_GRAD, i
    for a, b in zip(rays, rays_oo):
        assert rel_err(a.grad, b.grad) < TOL_GRAD


def test_strict_loss_grad_reruns_both_passes(cuda_dev):
    """Per-term upstream scales (strict_loss_grad): the re-run of both passes with the same draws
    equals the oracle's gradient of sum(scale_k * loss_k); the coarse pass takes the rgb and
    depth scales only."""
    from oracle import coslam_importance as CI
    N, R = 16, 1024
    ora, model = coslam_pair(cuda_dev, training_n_importance=N, strict_loss_grad=True)
    rays_o, rays_d, ts, td, noise = make_rays(R, seed=1)
    u = torch.rand(R, N, generator=torch.Generator().manual_seed(1))
    ro = rays_o.to(cuda_dev).requires_grad_(True)
    rd = rays_d.to(cuda_dev).requires_grad_(True)
    inp = dict(rays_o=ro, rays_d=rd, target_s=ts.to(cuda_dev), target_d=td.to(cuda_dev),
               first=True, noise=noise.to(cuda_dev), importance_u=u.to(cuda_dev))
    sc = (0.5, 2.0, 3.0, 0.25)
    out = model(inp)
    ld = model.get_loss_dict(out, inp, False, 0)
    sum(s * v for s, v in zip(sc, ld.values())).backward()
    torch.cuda.synchronize()
    rays_o.requires_grad_(True)
    rays_d.requires_grad_(True)
    _, ld_o, _ = CI.step(ora, rays_o, rays_d, ts, td, noise, u, z_fine=out['z_vals'].cpu())
    sum(s * v for s, v in zip(sc, ld_o.values())).backward()
    for i, (m, o) in enumerate(_weights(model, ora)):
        assert rel_err(m.grad, o.grad) < TOL_GRAD, i
    assert rel_err(ro.grad, rays_o.grad) < TOL_GRAD
    assert rel_err(rd.grad, rays_d.grad) < TOL_GRAD


def test_render_forward_only_with_depth(cuda_dev):
    from oracle import coslam_importance as CI
    N, R = 16, 2000
    ora, model = coslam_pair(cuda_dev, training_n_importance=N)
    rays_o, rays_d, ts, td, noise = make_rays(R, seed=4)
    u = torch.rand(R, N, generator=torch.Generator().manual_seed(4))
    with torch.no_grad():
        out = model.render_rays(rays_o.to(cuda_dev), rays_d.to(cuda_dev), target_d=td.to(cuda_dev),
                                noise=noise.to(cuda_dev), importance_u=u.to(cuda_dev))
        out_o = CI.render_rays(ora, rays_o, rays_d, td, noise, u, z_fine=out['z_vals'].cpu())
    torch.cuda.synchronize()
    for k in OUTS:
        assert max_abs(out[k], out_o[k]) < TOL_OUT, k
    assert max_abs(out['raw'], out_o['raw']) < 5e-5


def test_render_without_depth_raises(cuda_dev):
    """training_n_samples (256) + N samples per ray do not fit the fused kernels."""
    _, model = coslam_pair(cuda_dev, training_n_importance=16)
    rays_o, rays_d, _, _, _ = make_rays(8, seed=0)
    with torch.no_grad(), pytest.raises(ValueError, match='272 samples per ray.*at most 256'):
        model.render_rays(rays_o.to(cuda_dev), rays_d.to(cuda_dev))


def _build_algorithm(dev, seed, N, one_grid=True):
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
    cfg.model.training_n_importance = N
    cfg.model.oneGrid = one_grid
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


def _map(dev, graph, n_iters, N, one_grid, seed=11):
    random.seed(seed)
    algo, kfs, cur = _build_algorithm(dev, seed, N, one_grid)
    algo.config.graph_mapping = graph
    algo.config.min_sample_pixels = 256
    frames = kfs + [cur]
    torch.manual_seed(seed)
    losses = []
    if graph:
        algo.setup_optimizers(n_iters, frames, True)
        sess = algo.mapping_session(frames)
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


@pytest.mark.parametrize('one_grid', [True, False])
def test_graph_mapping_matches_generic_path(cuda_dev, one_grid):
    """The captured mapping iteration (coarse pass, importance step with u from the device seed,
    fine pass) equals the autograd iteration: the seed sequence is the same, so are the draws."""
    a_g, f_g, l_g = _map(cuda_dev, True, 7, 16, one_grid)
    a_e, f_e, l_e = _map(cuda_dev, False, 7, 16, one_grid)
    assert len(l_g) == len(l_e) == 7
    # the first iteration starts from the same state: the same jitter and importance draws give
    # the same loss up to the order of the reductions
    assert abs(l_g[0] - l_e[0]) <= 1e-5 * abs(l_e[0]), (l_g, l_e)
    for x, y in zip(l_g, l_e):
        assert abs(x - y) <= 2e-3 * abs(y), (l_g, l_e)
    assert l_g[-1] < l_g[0]
    # Adam steps an entry by about lr whatever its gradient's size, so entries whose gradient is
    # near zero amplify the atomic summation order over the iterations: an l2 bound, the one
    # the tables get (measured on an H100: 3.0e-3 for the first decoder layer with one grid)
    for p, q in zip(a_g.model.decoder.parameters(), a_e.model.decoder.parameters()):
        assert rel_err(p, q) < 1e-2
    assert rel_err(a_g.model.embed_fn.params, a_e.model.embed_fn.params) < 1e-2
    for fg, fe in zip(f_g, f_e):
        assert (fg.pose.data_t - fe.pose.data_t).abs().max() < 2e-5
        assert (fg.pose.data_r - fe.pose.data_r).abs().max() < 2e-5


def test_tracking_graph_matches_generic_iteration(cuda_dev):
    from xrdslam_b200.common import sample_window
    from xrdslam_b200.coslam_graph import TrackingGraphSession
    from xrdslam_b200.opt_pose import pose_matrices
    algo, kfs, cur = _build_algorithm(cuda_dev, 3, 16)
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


def test_run_and_eval_importance(cuda_dev, tmp_path):
    """A short synthetic Replica run with model.training_n_importance=16 through get_mesh and
    ds-eval."""
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
                      **REDUCED['co-slam'], **{'model.training_n_importance': 16})
    assert cfg.algorithm.model.training_n_importance == 16
    with warnings.catch_warnings():
        warnings.simplefilter('ignore', UserWarning)
        res = XRDSLAM(cfg).run()
    assert res['n_frames'] == N_FRAMES
    for name in ('eval.tar', 'final_mesh.ply', 'final_mesh_rec.ply'):
        assert os.path.exists(out / name), name
    m = EvalMatrics(output_dir=out, gt_mesh=gt, device=str(cuda_dev)).main()
    assert math.isfinite(float(m['accuracy'])) and math.isfinite(float(m['completion']))


# ---------------------------------------------------------------- float64 ---
def _f64_two_pass(refs, cand, amb, cand_sdfs):
    """oracle/coslam_f64.compare for a step of two passes: the float64 replays of the coarse and
    the fine pass (refs), their gradients and absolute-value bounds summed; a point ambiguous in
    either pass (a hidden unit near zero, or a ray whose first sdf sign change the candidate
    puts elsewhere) excludes what it touches, as compare() does for one pass."""
    from oracle.coslam_f64 import (RAY_KEYS, WEIGHT_KEYS, _ratio, abs_bounds, flip_bounds,
                                   level_slices, sdf_decision)
    dev = refs[0]['sdf'].device
    R = refs[0]['R']
    n_val = refs[0]['table'].numel()
    A, A_amb, g64 = {}, {}, {}
    drop_entry = torch.zeros(n_val, dtype=torch.bool, device=dev)
    drop_level = torch.zeros(n_val, dtype=torch.bool, device=dev)
    flip_rays = torch.zeros(R, dtype=torch.bool, device=dev)

    def touched_by(ref, points):
        t = torch.zeros(n_val // 2, dtype=torch.bool, device=dev)
        t[ref['idx'][points].reshape(-1)] = True
        return t.repeat_interleave(2)

    def add(d, k, v):
        d[k] = v if k not in d else d[k] + v
    for ref, sdf in zip(refs, cand_sdfs):
        S = ref['S']
        inds_c, _ = sdf_decision(sdf.detach().to(device=dev, dtype=torch.float32).reshape(R, S),
                                 ref['z'].float(), ref['trunc'])
        flip = inds_c != ref['inds']
        amb_b, pm = flip_bounds(ref, amb)
        fp = flip.repeat_interleave(S)
        if bool(fp.any()):
            A_fl = abs_bounds(ref, fp)
            amb_b = {k: v + A_fl[k] for k, v in amb_b.items()}
        for k, v in abs_bounds(ref).items():
            add(A, k, v)
        for k, v in amb_b.items():
            add(A_amb, k, v)
        for k, v in ref['grads'].items():
            add(g64, k, v)
        drop_entry |= touched_by(ref, pm | fp)
        drop_level |= touched_by(ref, fp)
        flip_rays |= flip
    rep = dict(n_flip_rays=int(flip_rays.sum()))
    g = cand['d_table'].detach().to(device=dev, dtype=torch.float64).reshape(-1)
    r = g64['d_table']
    lv, ent = [], []
    for a, b in level_slices(refs[0]['layout']):
        k = ~drop_level[a:b]
        lv.append(float((g[a:b][k] - r[a:b][k]).norm() / (r[a:b][k].norm() + 1e-300)))
        k = ~drop_entry[a:b]
        ent.append(_ratio((g[a:b] - r[a:b]).abs()[k], A['d_table'][a:b][k]))
    rep['level'], rep['entry_per_level'], rep['entry'] = lv, ent, max(ent)
    for key in WEIGHT_KEYS:
        err = (cand[key].detach().to(device=dev, dtype=torch.float64).reshape(-1) -
               g64[key].reshape(-1)).abs()
        rep[key] = _ratio(err, A[key].reshape(-1), A_amb[key].reshape(-1))
    for key in RAY_KEYS:
        gr = cand[key].detach().to(device=dev, dtype=torch.float64).reshape(R, 3)
        err = (gr - g64[key]).abs()[~flip_rays]
        den = (g64[key].abs() + A[key])[~flip_rays]
        rep[key] = _ratio(err, den, A_amb[key][~flip_rays])
    lc, lf = refs[0]['losses'], refs[1]['losses']
    want = torch.stack([lc[0] + lf[0], lc[1] + lf[1], lf[2], lf[3]])
    lo = cand['losses'].detach().to(device=dev, dtype=torch.float64).reshape(-1)
    rep['loss'] = float(((lo - want).abs() / want.abs().clamp_min(1e-12)).max())
    return rep


@pytest.mark.parametrize('N', [16, 53])
@pytest.mark.parametrize('kernel', [-1, -2])
@pytest.mark.parametrize('mode', [0, 1])
def test_step_vs_float64_per_entry(cuda_dev, N, kernel, mode):
    """Both passes against the float64 replay of oracle/coslam_f64.py, per hash level, per table
    entry, per weight element, per ray and per loss term, to the gates of
    test_coslam_grad_f64_gpu.py: the coarse pass replayed on its z_vals with loss scales
    (1, 1, 0, 0), the fine pass on the kernel's merged z_vals, the two summed."""
    from oracle.coslam_f64 import failures, replay_step
    from test_coslam_grad_f64_gpu import AMB, GATES
    R = 1024
    ora, model = coslam_pair(cuda_dev, training_n_importance=N, rays_per_tile=kernel,
                             precision=mode)
    ro, rd, ts, td, noise = make_rays(R, seed=R + N)
    u = torch.rand(R, N, generator=torch.Generator().manual_seed(N))
    dev = cuda_dev
    w = model._weights()
    out, g = model._launch(ro.to(dev), rd.to(dev), model.embed_fn.params, *w, ts.to(dev),
                           td.to(dev), noise.to(dev), with_grads=True, need_ray_grads=True,
                           importance_u=u.to(dev))
    # the coarse pass's sdf, for the sign-change decisions: the same pass forward only
    model.config.training_n_importance = 0
    try:
        oc, _ = model._launch(ro.to(dev), rd.to(dev), model.embed_fn.params, *w, ts.to(dev),
                              td.to(dev), noise.to(dev), with_grads=False)
    finally:
        model.config.training_n_importance = N
    torch.cuda.synchronize()
    with torch.no_grad():
        zc = ora.sample_z(R, td, noise)
    assert torch.equal(oc['z_vals'].cpu(), zc)
    zf = out['z_vals'].detach().cpu()
    refs = (replay_step(ora, ro, rd, ts, td, zc, loss_scale=(1., 1., 0., 0.), device=dev),
            replay_step(ora, ro, rd, ts, td, zf, device=dev))
    rep = _f64_two_pass(refs, dict(g, losses=out['losses']), AMB[mode],
                        (oc['raw'][..., 3], out['raw'][..., 3]))
    print(f'N={N} kernel={kernel} mode={mode}: entry {rep["entry"]:.3g} '
          f'level {max(rep["level"]):.3g} loss {rep["loss"]:.3g} flips {rep["n_flip_rays"]}')
    assert rep['n_flip_rays'] <= 2
    assert not failures(rep, GATES[mode]), failures(rep, GATES[mode])


# ---------------------------------------------------------------- sharding ---
def _dp_worker(rank, world, port, ret):
    """Mapping rays with importance sampling sharded over the ranks (generic autograd path, then
    the captured iteration) == the single-GPU step on the whole batch."""
    import os
    import sys
    import torch.distributed as dist
    here = os.path.dirname(os.path.abspath(__file__))
    sys.path.insert(0, here)
    sys.path.insert(0, os.path.dirname(here))
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    torch.cuda.set_device(rank)
    dev = torch.device('cuda', rank)
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=dev)
    from helpers import coslam_pair, make_rays, rel_err
    from test_coslam_importance_gpu import _build_algorithm
    from xrdslam_b200.dp import MappingDataParallel
    out = {}
    # ---- generic path: the fine pass's counts are all-reduced between importance and fine pass
    N, R = 16, 514
    _, model = coslam_pair(dev, training_n_importance=N)
    ro, rd, ts, td, noise = make_rays(R, seed=3)
    u = torch.rand(R, N, generator=torch.Generator().manual_seed(3))
    full = dict(rays_o=ro.to(dev), rays_d=rd.to(dev), target_s=ts.to(dev), target_d=td.to(dev),
                first=True, noise=noise.to(dev), importance_u=u.to(dev))
    params = [model.embed_fn.params] + list(model.decoder.parameters())
    keys = ('rgb_loss', 'depth_loss', 'sdf_loss', 'fs_loss')
    ld = model.get_loss_dict(model(full), full, True, 0)
    sum(ld.values()).backward()
    ref = [p.grad.clone() for p in params]
    ref_loss = torch.stack([ld[k].detach() for k in keys])
    for p in params:
        p.grad = None
    model.dp = dp = MappingDataParallel(params)
    sl = dp.shard(R)
    part = {k: (v[sl] if torch.is_tensor(v) else v) for k, v in full.items()}
    ld = model.get_loss_dict(model(part), part, True, 0)
    sum(ld.values()).backward()
    loss = torch.stack([ld[k].detach() for k in keys])
    dp.all_reduce_grads(extra=[loss])
    out['grad'] = max(rel_err(p.grad, g) for p, g in zip(params, ref))
    out['loss'] = float((loss - ref_loss).abs().max() / ref_loss.abs().max())

    # ---- captured iteration (training_perturb = 0: the coarse jitter and the importance draws
    # are keyed by the local ray index, the det draw and no jitter are not)
    def build(mapping_sample, with_dp):
        algo, kfs, cur = _build_algorithm(dev, 5, N)  # same seed: identical replicas
        algo.config.mapping_sample = mapping_sample
        algo.config.min_sample_pixels = mapping_sample
        algo.model.config.training_perturb = 0
        frames = kfs + [cur]
        if with_dp:
            ps = [algo.model.embed_fn.params] + list(algo.model.decoder.parameters())
            algo.model.dp = MappingDataParallel(ps)
        algo.setup_optimizers(4, frames, True)
        sess = algo.mapping_session(frames)
        sess._gen = torch.Generator().manual_seed(977)
        sess.begin(frames)
        return algo, frames, sess
    algo_s, frames_s, sess_s = build(4096, False)
    rows, ids = sess_s.make_resident_batch(frames_s)
    loss_s = float(sess_s.step_resident(0, (rows, ids)))
    algo_d, frames_d, sess_d = build(2048, True)
    assert sess_d.world == 2 and sess_d.R == 4096
    # one graph, or four segments around the three all-reduces if NCCL refused capture
    assert len(sess_d.graphs) == (1 if sess_d.single_graph else 4)
    sl = slice(rank * 4096, (rank + 1) * 4096)
    loss_d = float(sess_d.step_resident(0, (rows[sl].contiguous(), ids[sl].contiguous())))
    out['g_loss'] = abs(loss_d - loss_s) / abs(loss_s)
    out['g_table'] = rel_err(sess_d.grads[algo_d.model.embed_fn.params],
                             sess_s.grads[algo_s.model.embed_fn.params])
    out['g_decoder'] = max(rel_err(sess_d.grads[p], sess_s.grads[q]) for p, q in
                           zip(algo_d.model.decoder.parameters(), algo_s.model.decoder.parameters()))
    out['g_d_rot'] = rel_err(sess_d.d_rot_it, sess_s.d_rot_it)
    ret[rank] = out
    sess_d.release()
    sess_s.release()
    torch.cuda.synchronize()
    dist.barrier()
    dist.destroy_process_group()


def test_sharded_mapping_with_importance_equals_single_gpu():
    """Gates of test_dp_gpu.py."""
    import os
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < 2:
        pytest.skip('needs 2 GPUs')
    world = 2
    ret = mp.Manager().dict()
    mp.spawn(_dp_worker, args=(world, 33500 + (os.getpid() % 2000), ret), nprocs=world, join=True)
    print(dict(ret))
    for r in range(world):
        o = ret[r]
        assert o['grad'] < 1e-4 and o['loss'] < 1e-5, o
        assert o['g_loss'] < 1e-5 and o['g_table'] < 1e-4 and o['g_decoder'] < 1e-4, o
        assert o['g_d_rot'] < 1e-3, o


class _ThreadDP:
    """Two ranks as two threads on one GPU: all_reduce_sum adds the ranks' tensors, in rank
    order on both.  What JointEncoding._launch needs of xrdslam_b200.dp.MappingDataParallel."""
    def __init__(self, rank, box, barrier):
        self.rank, self.world, self.box, self.barrier = rank, 2, box, barrier

    def all_reduce_sum(self, t):
        torch.cuda.synchronize()
        self.box[self.rank] = t.clone()
        self.barrier.wait()
        total = self.box[0] + self.box[1]
        self.barrier.wait()
        return t.copy_(total)


def test_sharded_generic_mapping_with_importance_on_one_gpu(cuda_dev):
    """The sharded generic path (coarse counts all-reduce, importance, fine counts all-reduce,
    n_rays_global of the fine pass) with its two ranks as threads on this GPU: the ranks'
    summed gradients and loss terms equal the single-GPU step on the whole batch."""
    import threading
    N, R = 16, 514
    _, single = coslam_pair(cuda_dev, training_n_importance=N)
    ro, rd, ts, td, noise = make_rays(R, seed=3)
    u = torch.rand(R, N, generator=torch.Generator().manual_seed(3))
    full = dict(rays_o=ro.to(cuda_dev), rays_d=rd.to(cuda_dev), target_s=ts.to(cuda_dev),
                target_d=td.to(cuda_dev), first=True, noise=noise.to(cuda_dev),
                importance_u=u.to(cuda_dev))
    keys = ('rgb_loss', 'depth_loss', 'sdf_loss', 'fs_loss')

    def params(m):
        return [m.embed_fn.params] + list(m.decoder.parameters())
    ld = single.get_loss_dict(single(full), full, True, 0)
    sum(ld.values()).backward()
    ref_loss = torch.stack([ld[k].detach() for k in keys])
    ranks = [coslam_pair(cuda_dev, training_n_importance=N)[1] for _ in range(2)]
    box, barrier, res, errs = {}, threading.Barrier(2), {}, []

    def run(rank):
        try:
            m = ranks[rank]
            m.dp = _ThreadDP(rank, box, barrier)
            sl = slice(rank * R // 2, (rank + 1) * R // 2)
            part = {k: (v[sl] if torch.is_tensor(v) else v) for k, v in full.items()}
            ld_r = m.get_loss_dict(m(part), part, True, 0)
            sum(ld_r.values()).backward()
            torch.cuda.synchronize()
            res[rank] = torch.stack([ld_r[k].detach() for k in keys])
        except BaseException as e:  # noqa: B902 -- re-raised in the test's thread
            errs.append(e)
            barrier.abort()
    th = [threading.Thread(target=run, args=(r,)) for r in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    if errs:
        raise errs[0]
    loss = res[0] + res[1]
    assert float((loss - ref_loss).abs().max() / ref_loss.abs().max()) < 1e-5
    for p0, p1, q in zip(params(ranks[0]), params(ranks[1]), params(single)):
        assert rel_err(p0.grad + p1.grad, q.grad) < 1e-4
