"""The restatements of oracle/frontend_f64.py, on the CPU: the float64 pose-chain references
against torch float64 autograd and central differences, adam_f32 against torch.optim.Adam and
against its own rule in float64."""
import numpy as np
import pytest
import torch

from oracle import frontend_f64 as F
from xrdslam_b200.opt_pose import OptimizablePose

THETAS = [1e-6, 1e-4, 1e-2, 0.5, 2.0, np.pi - 1e-3, np.pi, 3.5, 7.0]


def _rot(thetas, seed):
    g = np.random.default_rng(seed)
    a = g.normal(size=(len(thetas), 3))
    return a / np.linalg.norm(a, axis=1, keepdims=True) * np.asarray(thetas)[:, None]


class _Rodrigues(torch.autograd.Function):
    """rodrigues_f64 with rodrigues_bwd_f64 as its backward, for gradcheck."""
    @staticmethod
    def forward(ctx, rot, trans):
        ctx.save_for_backward(rot)
        return torch.from_numpy(F.rodrigues_f64(rot.detach().numpy(), trans.detach().numpy()))

    @staticmethod
    def backward(ctx, G):
        rot, = ctx.saved_tensors
        d_rot, d_trans = F.rodrigues_bwd_f64(rot.numpy(), G.numpy())
        return torch.from_numpy(d_rot), torch.from_numpy(d_trans)


def test_rodrigues_f64_matches_optimizable_pose():
    rot = _rot(THETAS, 0)
    trans = np.random.default_rng(1).normal(size=rot.shape)
    M = F.rodrigues_f64(rot, trans)
    for i in range(len(rot)):
        R = OptimizablePose.axis_angle_to_rotation_matrix(torch.from_numpy(rot[i])).numpy()
        assert np.abs(M[i, :3, :3] - R).max() < 1e-14
        assert np.array_equal(M[i, :3, 3], trans[i]) and np.array_equal(M[i, 3], [0, 0, 0, 1])
    assert np.array_equal(F.rodrigues_f64(np.array([[1e-9, 0, 0]]), np.zeros((1, 3)))[0],
                          np.eye(4))


def test_rodrigues_bwd_f64_gradcheck():
    rot = torch.from_numpy(_rot(THETAS, 2)).requires_grad_(True)
    trans = torch.randn(len(THETAS), 3, dtype=torch.float64, generator=torch.Generator().manual_seed(3))
    trans.requires_grad_(True)
    assert torch.autograd.gradcheck(_Rodrigues.apply, (rot, trans), eps=1e-7, atol=1e-7, rtol=1e-6)


def test_rodrigues_bwd_f64_matches_autograd_and_central_differences():
    rot = _rot(THETAS, 4)
    G = np.random.default_rng(5).normal(size=(len(THETAS), 4, 4))
    d_rot, d_trans = F.rodrigues_bwd_f64(rot, G)
    assert np.array_equal(d_trans, G[:, :3, 3])
    for i in range(len(rot)):
        w = torch.from_numpy(rot[i].copy()).requires_grad_(True)
        (OptimizablePose.axis_angle_to_rotation_matrix(w) * torch.from_numpy(G[i, :3, :3])).sum().backward()
        # torch's 1 - cos(th) cancels in float64 too: ~1e-16 / th
        assert np.abs(d_rot[i] - w.grad.numpy()).max() <= 1e-9 * np.abs(G[i]).sum()
        h = 1e-6 * max(1.0, THETAS[i])
        for d in range(3):
            e = np.zeros((1, 3))
            e[0, d] = h
            f = lambda r: (F.rodrigues_f64(r, np.zeros((1, 3)))[0] * G[i]).sum()
            cd = (f(rot[i:i + 1] + e) - f(rot[i:i + 1] - e)) / (2 * h)
            assert abs(cd - d_rot[i, d]) <= 1e-7 * np.abs(G[i]).sum(), (THETAS[i], d)
    fixed = np.zeros(len(rot), np.uint8)
    fixed[[0, -1]] = 1
    d_rot_f, d_trans_f = F.rodrigues_bwd_f64(rot, G, fixed)
    assert not d_rot_f[[0, -1]].any() and not d_trans_f[[0, -1]].any()
    assert np.array_equal(d_rot_f[1:-1], d_rot[1:-1])
    # identity branch: no rotation gradient at or below 1e-8
    assert not F.rodrigues_bwd_f64(np.array([[0.0, 0, 0], [5e-9, 0, 0]]), G[:2])[0].any()


@pytest.mark.parametrize('n_poses', [1, 5, 70])
def test_rays_bwd_f64_matches_index_put_autograd(n_poses):
    g = torch.Generator().manual_seed(n_poses)
    R = 600
    dirs = torch.randn(R, 3, generator=g, dtype=torch.float64)
    ids = torch.randint(-n_poses, n_poses + 3, (R,), generator=g)   # some out of range
    d_o = torch.randn(R, 3, generator=g, dtype=torch.float64)
    d_d = torch.randn(R, 3, generator=g, dtype=torch.float64)
    live = (ids >= -n_poses) & (ids < n_poses)
    row = torch.where(ids < 0, ids + n_poses, ids)[live]
    P = torch.zeros(n_poses, 4, 4, dtype=torch.float64, requires_grad=True)
    M = P[row]   # backward: index_put(accumulate=True)
    rd = (dirs[live, None, :] * M[:, :3, :3]).sum(-1)
    ((rd * d_d[live]).sum() + (M[:, :3, 3] * d_o[live]).sum()).backward()
    dp, abs_sum, n_p = F.rays_bwd_f64(dirs.numpy(), ids.numpy(), n_poses, d_o.numpy(), d_d.numpy())
    assert np.abs(dp - P.grad.numpy()).max() <= 1e-13 * abs_sum.max()
    assert not dp[:, 3].any() and not abs_sum[:, 3].any()
    assert np.array_equal(n_p, np.bincount(row.numpy(), minlength=n_poses))
    # each gradient alone
    dp_o, _, _ = F.rays_bwd_f64(dirs.numpy(), ids.numpy(), n_poses, d_o.numpy(), None)
    dp_d, _, _ = F.rays_bwd_f64(dirs.numpy(), ids.numpy(), n_poses, None, d_d.numpy())
    assert not dp_o[:, :3, :3].any() and not dp_d[:, :3, 3].any()
    assert np.allclose(dp_o + dp_d, dp, rtol=0, atol=1e-12)


def test_rays_fwd_f32_matches_torch():
    g = torch.Generator().manual_seed(0)
    dirs = torch.randn(300, 3, generator=g)
    poses = torch.randn(4, 4, 4, generator=g)
    ids = torch.randint(-4, 4, (300,), generator=g)
    ro, rd = F.rays_fwd_f32(dirs.numpy(), ids.numpy(), poses.numpy())
    P = poses.double()[ids]
    assert np.abs(rd - (dirs.double()[:, None, :] * P[:, :3, :3]).sum(-1).numpy()).max() < 1e-5
    assert np.array_equal(ro, poses[ids, :3, 3].numpy())
    ro, rd = F.rays_fwd_f32(dirs.numpy()[:2], np.array([4, -5]), poses.numpy())
    assert np.isnan(ro).all() and np.isnan(rd).all()


ADAM_CASES = [dict(lr=1e-2, eps=1e-15, betas=(0.9, 0.99), weight_decay=0.0),
              dict(lr=1e-3, eps=1e-8, betas=(0.9, 0.999), weight_decay=1e-2)]


def _one_minus_beta_gap(beta):
    """Relative gap between the kernel's 1 - beta (float32 arithmetic on float32(beta)) and
    torch's (python double, then float32): 4 u for 0.9, 16 u for 0.99, 216 u for 0.999."""
    f = np.float32
    return abs(float(f(1) - f(beta)) - float(f(1 - beta))) / (1 - beta)


@pytest.mark.parametrize('kw', ADAM_CASES)
def test_adam_f32_matches_torch_adam(kw):
    """Torch forms 1 - beta in double where the kernel subtracts in float32, divides by
    sqrt(bc2) where the kernel multiplies by its reciprocal, and lerps / addcmuls with its own
    roundings.  So m and v differ by the 1 - beta gap plus a few u, and each step's update
    (|update| <= lr) by at most lr (gap1 + gap2 + 16 u) plus one rounding of p."""
    g = torch.Generator().manual_seed(7)
    p0 = torch.randn(4099, generator=g)
    p_t = p0.clone().requires_grad_(True)
    opt = torch.optim.Adam([p_t], foreach=False, **kw)
    p, m, v = p0.numpy().copy(), np.zeros(4099, np.float32), np.zeros(4099, np.float32)
    b1, b2 = kw['betas']
    gap1, gap2 = _one_minus_beta_gap(b1), _one_minus_beta_gap(b2)
    for t in range(1, 13):
        gr = torch.randn(4099, generator=g) * (0.0 if t == 4 else 1.0)
        p_t.grad = gr.clone()
        opt.step()
        p, _, m, v = F.adam_f32(p, gr.numpy(), m, v, kw['lr'], b1, b2, kw['eps'], kw['weight_decay'],
                                1 - b1 ** t, 1 - b2 ** t)
        st = opt.state[p_t]
        pt = p_t.detach().numpy()
        tol = t * (np.spacing(np.abs(pt)) + kw['lr'] * (gap1 + gap2 + 16 * F.U32))
        assert (np.abs(p - pt) <= tol).all(), t
        assert np.abs(m - st['exp_avg'].numpy()).max() <= (gap1 + 4 * F.U32) * np.abs(m).max()
        assert np.abs(v - st['exp_avg_sq'].numpy()).max() <= (gap2 + 4 * F.U32) * np.abs(v).max()


@pytest.mark.parametrize('kw', ADAM_CASES)
def test_adam_f32_near_float64_rule(kw):
    """Away from underflow fp32 stays within a few u per step of the float64 rule: per step
    |dp| <= u |p| + ~8 u |update|, over 12 steps and |update| <= lr (Adam's step bound)."""
    g = np.random.default_rng(8)
    p32 = g.normal(size=2000).astype(np.float32)
    p64, m32, v32 = p32.astype(np.float64), np.zeros(2000, np.float32), np.zeros(2000, np.float32)
    m64, v64 = np.zeros(2000), np.zeros(2000)
    b1, b2 = kw['betas']
    for t in range(1, 13):
        gr = g.normal(size=2000).astype(np.float32)
        args = (kw['lr'], b1, b2, kw['eps'], kw['weight_decay'], 1 - b1 ** t, 1 - b2 ** t)
        p32, _, m32, v32 = F.adam_f32(p32, gr, m32, v32, *args)
        p64, m64, v64 = F.adam_f64(p64, gr, m64, v64, *args)
        tol = t * F.U32 * (np.abs(p64) + 16 * kw['lr']) + 1e-6 * kw['lr'] * t
        assert (np.abs(p32 - p64) <= tol).all(), t


def test_adam_f32_mask_zero_grad_dyn():
    g = np.random.default_rng(9)
    p, gr = g.normal(size=18).astype(np.float32), g.normal(size=18).astype(np.float32)
    m, v = g.normal(size=18).astype(np.float32), np.abs(g.normal(size=18)).astype(np.float32)
    mask = np.array([1, 0, 1, 0, 0, 1], np.uint8)
    args = (1e-2, 0.9, 0.99, 1e-15, 0.0, 0.1, 0.01)
    p1, g1, m1, v1 = F.adam_f32(p, gr, m, v, *args, row_mask=mask, row_len=3, zero_grad=1)
    full = F.adam_f32(p, gr, m, v, *args)
    live = np.repeat(mask.astype(bool), 3)
    assert not g1.any()
    for a, b, c in ((p1, full[0], p), (m1, full[2], m), (v1, full[3], v)):
        assert np.array_equal(a[live], b[live]) and np.array_equal(a[~live], c[~live])
    dyn = F.adam_f32(p, gr, m, v, 5.0, 0.9, 0.99, 1e-15, 0.0, 9.0, 9.0, dyn=args[:1] + args[-2:])
    assert all(np.array_equal(a, b) for a, b in zip(dyn, full))
