"""The camera-pose chain and the fused Adam step on the device, bit for bit or within derived
float64 bounds (oracle/frontend_f64.py):

- xrd_rays_from_poses: rays_d bit for bit against rays_fwd_f32, rays_o the pose column; NaN
  rays for out-of-range ids.
- xrd_rays_pose_grads: every entry within gamma(n_p + 2) * sum|term| of the float64 sum, which
  holds for any summation order (the atomics reorder it from run to run); entries no ray
  reaches exactly 0.  Shapes cover the warp-uniform shuffle path (frame-major ids, a frame
  boundary inside a warp, at n_poses on both sides of the shared-memory limit MAXP = 64 with
  every pose row, the highest ones included, reduced by whole warps), the per-lane fallback
  (random or scattered ids, lane 0 out of range) on both sides of MAXP, and more rays than
  one grid-stride pass covers.
- xrd_pose_matrices / _grads against the float64 Rodrigues:
    forward   |R - R64| <= (C1 + C2 th) u for every entry (|R|, |K|, |K^2| <= 1).  k = w / th
              carries <= 3 u (the three-term sum of squares and its sqrt 2 u, the division u),
              K^2 <= 8 u, sinf / cosf <= 2 ulp each, c1 = 2 sin^2(th / 2) <= 8 u relative, and
              the rounding of th (<= 2 u th) moves R by |dR/dth| <= 2 per unit: 2 + 3 + 8 + 2
              -> C1 = 16 with room, C2 = 4.
    backward  |d_rot - (old + g64)| <= u |old + g64| + C u ||G||_F (1 + th): each of dK, dk,
              <G,K>, <G,K^2> is a sum of <= 6 products of |G| entries with |K| <= 1 at <= 8 u
              each, the projection / th divides an O(th ||G||) quantity whose rounding is
              O(u th ||G||) (c1 = 2 sin^2(th / 2) keeps its relative error at the small angles
              where 1 - cosf(th) cancels to 0), and the th rounding adds 2 u th ||G|| per
              unit of |d g / d th| <= 2 -> C = 32.
    d_trans = fl(old + G[:3, 3]) bit for bit; fixed rows and identity-branch rows untouched.
- xrd_adam_step bit for bit against adam_f32 (param, exp_avg, exp_avg_sq and grad after the
  call), 12 chained steps.
- The Co-SLAM tracking and mapping graph sessions: the session's d_rot / d_trans against the
  float64 chain of its own ray gradients (the ray bound carried through the exact |d g / d G|
  of the Rodrigues backward, plus the pose bound), and its pose Adam step bit for bit.

Mutations of the kernel outputs that a faulty kernel would produce must fail the same bounds.
test_report_worst prints the worst error / bound ratio of every check.
"""
import numpy as np
import pytest
import torch

from oracle import frontend_f64 as F

U = F.U32
C1, C2, C_BWD = 16.0, 4.0, 32.0
THETAS = [0.0, 1e-9, 2e-8, 1e-6, 1e-4, 1e-2, 0.5, np.pi - 1e-3, np.pi, 3.5, 7.0]
SEEN = {}   # check -> worst error / bound ratio


def _note(key, err, bound):
    err, bound = np.asarray(err, np.float64), np.asarray(bound, np.float64)
    assert ((bound > 0) | (err == 0)).all(), f'{key}: an entry with a zero bound is not exact'
    r = float((err / np.where(bound > 0, bound, 1.0)).max()) if err.size else 0.0
    SEEN[key] = max(SEEN.get(key, 0.0), r)
    return r


def _bits(a):
    return np.ascontiguousarray(np.asarray(a, np.float32)).view(np.int32)


def _ptr(t):
    return None if t is None else t.data_ptr()


def _launch(dev, name, *args):
    from xrdslam_b200 import _cabi
    _cabi.launch_on(dev, name, *args)
    torch.cuda.synchronize(dev)


# ------------------------------------------------------------------ rays forward ---
@pytest.mark.gpu
@pytest.mark.parametrize('R', [1, 31, 32, 33, 5000])
@pytest.mark.parametrize('ids_kind', ['null', 'negative', 'out_of_range'])
def test_rays_from_poses_bit_exact(cuda_dev, R, ids_kind):
    g = torch.Generator().manual_seed(R)
    n = 5
    dirs = torch.randn(R, 3, generator=g)
    poses = torch.randn(n, 4, 4, generator=g)
    ids = {'null': None, 'negative': torch.randint(-n, 0, (R,), generator=g),
           'out_of_range': torch.randint(-n - 2, n + 2, (R,), generator=g)}[ids_kind]
    if ids is not None and ids_kind == 'out_of_range':
        ids[0] = n   # at least one
    d = lambda t: None if t is None else t.to(cuda_dev).contiguous()
    ro, rd = torch.empty(R, 3, device=cuda_dev), torch.empty(R, 3, device=cuda_dev)
    dev_in = [d(dirs), d(ids), d(poses)]   # held until the launch has run
    _launch(cuda_dev, 'xrd_rays_from_poses', R, *map(_ptr, dev_in), n, _ptr(ro), _ptr(rd))
    ro_ref, rd_ref = F.rays_fwd_f32(dirs.numpy(), None if ids is None else ids.numpy(),
                                    poses.numpy())
    assert np.array_equal(_bits(ro.cpu()), _bits(ro_ref))
    assert np.array_equal(_bits(rd.cpu()), _bits(rd_ref))
    if ids_kind == 'out_of_range':
        assert np.isnan(rd.cpu().numpy()[0]).all()


# ------------------------------------------------------------------ rays backward ---
def _frame_major(n_poses, per_frame):
    return torch.arange(n_poses).repeat_interleave(per_frame)


def _rays_case(name, sms):
    """-> (R, n_poses, ids or None, use d_o, use d_d)"""
    g = torch.Generator().manual_seed(len(name))
    if name == 'frames257':         # sample_window layout: frame boundaries inside warps
        return 5 * 257, 5, _frame_major(5, 257), True, True
    if name == 'same_id':
        return 5000, 4, torch.full((5000,), 2, dtype=torch.int64), True, True
    if name == 'random':
        return 5000, 6, torch.randint(-6, 8, (5000,), generator=g), True, True
    if name == 'lane0_out_of_range':   # every other warp: lane 0 dead -> per-lane fallback
        ids = _frame_major(3, 1400)
        ids[::64] = 9
        return ids.numel(), 3, ids, True, True
    if name.startswith('n_poses'):
        n = int(name[7:])
        ids = torch.sort(torch.randint(0, n, (4000,), generator=g))[0]
        ids[1::7] = torch.randint(-n, n, (ids[1::7].numel(),), generator=g)   # some scattered
        return 4000, n, ids, True, True
    if name.startswith('uniform'):   # frame-major, 77 rays per frame (not a multiple of 32), the
        n = int(name[7:])              # last frame addressed as -1 like the mapping batch's current
        ids = _frame_major(n, 77)      # frame: uniform warps at every pose row, above MAXP too
        ids[-77:] = -1
        return ids.numel(), n, ids, True, True
    if name == 'grid_stride':       # more rays than one pass of num_SMs blocks x 256 threads
        R = sms * 256 * 3 + 77
        return R, 8, torch.sort(torch.randint(0, 8, (R,), generator=g))[0], True, True
    if name == 'only_d_o':
        return 3000, 3, _frame_major(3, 1000), True, False
    if name == 'only_d_d':
        return 3000, 3, _frame_major(3, 1000), False, True
    if name == 'null_ids':
        return 2000, 1, None, True, True
    if name == 'R0':
        return 0, 4, torch.zeros(0, dtype=torch.int64), True, True
    raise KeyError(name)


RAYS_CASES = ['frames257', 'same_id', 'random', 'lane0_out_of_range', 'n_poses1', 'n_poses63',
              'n_poses64', 'n_poses65', 'n_poses100', 'uniform63', 'uniform64', 'uniform65',
              'uniform100', 'grid_stride', 'only_d_o', 'only_d_d',
              'null_ids', 'R0']


def _rays_bwd(dev, name):
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    R, n, ids, use_o, use_d = _rays_case(name, sms)
    g = torch.Generator().manual_seed(R + n)
    dirs = torch.randn(R, 3, generator=g)
    d_o = torch.randn(R, 3, generator=g) if use_o else None
    d_d = torch.randn(R, 3, generator=g) if use_d else None
    if ids is not None:   # rays with an out-of-range id must not be read
        row, live = F.pose_rows(ids.numpy(), R, n)
        dead = torch.from_numpy(~live)
        for t in (d_o, d_d):
            if t is not None:
                t[dead] = float('nan')
    d = lambda t: None if t is None else t.to(dev).contiguous()
    out = torch.full((n, 4, 4), float('nan'), device=dev)   # overwritten: "zeroed inside"
    dirs_d, ids_d, d_o_d, d_d_d = (d(t) if R else None for t in (dirs, ids, d_o, d_d))
    _launch(dev, 'xrd_rays_pose_grads', R, _ptr(dirs_d), _ptr(ids_d), n, _ptr(d_o_d), _ptr(d_d_d),
            _ptr(out))
    ref, A, n_p = F.rays_bwd_f64(dirs.numpy(), None if ids is None else ids.numpy(), n,
                                 None if d_o is None else d_o.numpy(),
                                 None if d_d is None else d_d.numpy())
    bound = F.gamma(n_p + 2)[:, None, None] * A
    return out.cpu().double().numpy(), ref, bound, dict(dirs=dirs, ids=ids, d_o=d_o, d_d=d_d, n=n)


def _uniform_warps(ids, R, n):
    """-> {warp: pose row} of the warps k_bwd reduces with the shuffle (every in-range lane on
    lane 0's row, lane 0 in range); warps start at multiples of 32 of the ray index."""
    row, live = F.pose_rows(None if ids is None else ids.numpy(), R, n)
    out = {}
    for w in range(0, R, 32):
        r, lv = row[w:w + 32], live[w:w + 32]
        if lv[0] and (r[lv] == r[0]).all():
            out[w // 32] = int(r[0])
    return out


def _rays_fails(cand, ref, bound):
    return not (np.abs(cand - ref) <= bound).all()


@pytest.mark.gpu
@pytest.mark.parametrize('case', RAYS_CASES)
def test_rays_pose_grads_within_order_free_bound(cuda_dev, case):
    out, ref, bound, inp = _rays_bwd(cuda_dev, case)
    assert np.isfinite(out).all()
    assert not out[:, 3].any(), 'bottom row'
    r = _note(f'rays_bwd {case}', np.abs(out - ref), bound)
    assert r <= 1.0, (case, r)
    if case.startswith('uniform'):   # the shuffle path ran, into global memory above MAXP
        rows = set(_uniform_warps(inp['ids'], inp['ids'].numel(), inp['n']).values())
        assert rows == set(range(inp['n']))
    if case == 'R0':
        assert not out.any()


def _ray_terms(inp, r):
    dirs, d_o, d_d = (inp[k] for k in ('dirs', 'd_o', 'd_d'))
    t = np.zeros((4, 4))
    t[:3, :3] = d_d[r].double().numpy()[:, None] * dirs[r].double().numpy()[None, :]
    t[:3, 3] = d_o[r].double().numpy()
    return t


@pytest.mark.gpu
def test_mutation_rays_drop_largest_ray_of_one_pose(cuda_dev):
    out, ref, bound, inp = _rays_bwd(cuda_dev, 'frames257')
    rows = np.nonzero(inp['ids'].numpy() == 2)[0]
    r = rows[np.argmax([np.abs(_ray_terms(inp, q)).sum() for q in rows])]
    mut = out.copy()
    mut[2] -= _ray_terms(inp, r)
    assert _rays_fails(mut, ref, bound)


@pytest.mark.gpu
def test_mutation_rays_warp_boundary_ray_moved_to_neighbour_pose(cuda_dev):
    """Ray 256 (lane 0 of warp 8, the last ray of frame 0) credited to frame 1, whose rays
    start at lane 1 of the same warp."""
    out, ref, bound, inp = _rays_bwd(cuda_dev, 'frames257')
    assert int(inp['ids'][256]) == 0 and int(inp['ids'][257]) == 1
    t = _ray_terms(inp, 256)
    mut = out.copy()
    mut[0] -= t
    mut[1] += t
    assert _rays_fails(mut, ref, bound)


@pytest.mark.gpu
@pytest.mark.parametrize('case', ['uniform63', 'uniform100'])
def test_mutation_rays_uniform_warp_row_stride_12(cuda_dev, case):
    """Every shuffle-reduced warp sum added at id0 * 12 + k instead of id0 * 16 + k (the
    12-float stride of the shared accumulator used for the [n,4,4] output)."""
    out, ref, bound, inp = _rays_bwd(cuda_dev, case)
    R, n = inp['ids'].numel(), inp['n']
    mut = out.reshape(-1).copy()
    for w, row in _uniform_warps(inp['ids'], R, n).items():
        t = sum(_ray_terms(inp, q) for q in range(32 * w, min(32 * w + 32, R))).reshape(-1)[:12]
        mut[row * 16:row * 16 + 12] -= t
        mut[row * 12:row * 12 + 12] += t
    assert _rays_fails(mut.reshape(out.shape), ref, bound)


@pytest.mark.gpu
def test_mutation_rays_outer_product_transposed(cuda_dev):
    out, ref, bound, _ = _rays_bwd(cuda_dev, 'frames257')
    mut = out.copy()
    mut[:, :3, :3] = np.swapaxes(out[:, :3, :3], 1, 2)
    assert _rays_fails(mut, ref, bound)


# ------------------------------------------------------------------ poses ---
def _rot_table(n, seed):
    """n axis-angle rows cycling through THETAS x (random axis, +-e0, +-e1, +-e2)."""
    g = np.random.default_rng(seed)
    axes = [None] + [s * np.eye(3)[i] for i in range(3) for s in (1, -1)]
    rows = []
    for i in range(n):
        th = THETAS[i % len(THETAS)]
        a = axes[(i // len(THETAS)) % len(axes)]
        if a is None:
            a = g.normal(size=3)
            a /= np.linalg.norm(a)
        rows.append(a * th)
    return np.asarray(rows).astype(np.float32)


def _pose_run(dev, n, seed=0):
    g = np.random.default_rng(seed + n)
    rot = _rot_table(n, seed)
    if n >= len(THETAS) * 7:
        rot[len(THETAS) * 7:] = (g.normal(size=(n - len(THETAS) * 7, 3)) *
                                 g.choice([1e-4, 0.3, 2.0, 5.0], size=(n - len(THETAS) * 7, 1)))
    trans = g.normal(size=(n, 3)).astype(np.float32)
    G = g.normal(size=(n, 4, 4)).astype(np.float32)
    old_r = g.normal(size=(n, 3)).astype(np.float32)
    old_t = g.normal(size=(n, 3)).astype(np.float32)
    fixed = np.zeros(n, np.uint8)
    if n > 2:
        fixed[[0, n - 1, n // 2]] = 1
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    rot_d, trans_d, G_d, fixed_d = d(rot), d(trans), d(G), d(fixed) if n > 2 else None
    M = torch.empty(n, 4, 4, device=dev)
    _launch(dev, 'xrd_pose_matrices', n, _ptr(rot_d), _ptr(trans_d), _ptr(M))
    d_rot, d_trans = d(old_r), d(old_t)
    _launch(dev, 'xrd_pose_matrices_grads', n, _ptr(rot_d), _ptr(G_d), _ptr(fixed_d), _ptr(d_rot),
            _ptr(d_trans))
    return dict(rot=rot, trans=trans, G=G, old_r=old_r, old_t=old_t, fixed=fixed,
                M=M.cpu().numpy(), d_rot=d_rot.cpu().numpy(), d_trans=d_trans.cpu().numpy())


def _pose_bwd_bound(rot, G, ref_total):
    th = np.linalg.norm(rot.astype(np.float64), axis=1)
    gn = np.linalg.norm(G[:, :3, :3].astype(np.float64), axis=(1, 2))
    return U * np.abs(ref_total) + (C_BWD * U * gn * (1 + th))[:, None]


@pytest.mark.gpu
@pytest.mark.parametrize('n', [1, 64, 65, 1000])
def test_pose_matrices_within_bound(cuda_dev, n):
    o = _pose_run(cuda_dev, n)
    ref = F.rodrigues_f64(o['rot'], o['trans'])
    th = np.linalg.norm(o['rot'].astype(np.float64), axis=1)
    err = np.abs(o['M'][:, :3, :3] - ref[:, :3, :3])
    _note('pose_fwd', err, np.broadcast_to(((C1 + C2 * th) * U)[:, None, None], err.shape))
    assert (err <= ((C1 + C2 * th) * U)[:, None, None]).all()
    assert np.array_equal(_bits(o['M'][:, :3, 3]), _bits(o['trans']))
    assert np.array_equal(o['M'][:, 3], np.tile([0, 0, 0, 1], (n, 1)))
    ident = th <= F.THETA_EPS
    assert np.array_equal(o['M'][ident, :3, :3], np.broadcast_to(np.eye(3), (ident.sum(), 3, 3)))


@pytest.mark.gpu
@pytest.mark.parametrize('n', [1, 64, 65, 1000])
def test_pose_grads_within_bound(cuda_dev, n):
    o = _pose_run(cuda_dev, n)
    fixed = o['fixed'].astype(bool)
    ref, ref_t = F.rodrigues_bwd_f64(o['rot'], o['G'], fixed)
    total = o['old_r'].astype(np.float64) + ref
    bound = _pose_bwd_bound(o['rot'], o['G'], total)
    err = np.abs(o['d_rot'] - total)
    live = ~fixed
    r = _note('pose_bwd', err[live], bound[live])
    assert r <= 1.0, r
    # fixed rows untouched, d_trans = fl(old + G[:3, 3]) bit for bit, identity rows keep d_rot
    assert np.array_equal(_bits(o['d_rot'][fixed]), _bits(o['old_r'][fixed]))
    assert np.array_equal(_bits(o['d_trans'][fixed]), _bits(o['old_t'][fixed]))
    assert np.array_equal(_bits(o['d_trans'][live]), _bits(o['old_t'][live] + o['G'][live, :3, 3]))
    ident = live & (np.linalg.norm(o['rot'].astype(np.float64), axis=1) <= F.THETA_EPS)
    assert ident.any() and np.array_equal(_bits(o['d_rot'][ident]), _bits(o['old_r'][ident]))


@pytest.mark.gpu
@pytest.mark.parametrize('fault', [dict(project=False), dict(thresh=1e-7),
                                   dict(transpose_k=False)])
def test_mutation_pose_grads(cuda_dev, fault):
    """The kernel's output moved by what the fault changes in float64 fails the bound."""
    o = _pose_run(cuda_dev, 65)
    fixed = o['fixed'].astype(bool)
    ref, _ = F.rodrigues_bwd_f64(o['rot'], o['G'], fixed)
    mut, _ = F.rodrigues_bwd_f64(o['rot'], o['G'], fixed, **fault)
    total = o['old_r'].astype(np.float64) + ref
    cand = o['d_rot'].astype(np.float64) + (mut - ref)
    assert not (np.abs(cand - total) <= _pose_bwd_bound(o['rot'], o['G'], total)).all()


# ------------------------------------------------------------------ Adam ---
def _adam_steps(dev, specs, zero_grad=0, steps=12, seed=0):
    """Run `steps` chained xrd_adam_step calls over the tensors of `specs` and hold every output
    to adam_f32 bit for bit.  spec keys: n, misalign, row_len (row mask), wd, dyn, gscale,
    lr, betas, eps."""
    from xrdslam_b200 import _cabi
    from xrdslam_b200.optimizers import adam_desc
    g = np.random.default_rng(seed)
    T, H = [], []
    for s in specs:
        n, off = s['n'], int(s.get('misalign', False))
        # at least one element: an empty view's data_ptr() is NULL, which the entry rejects
        bufs = [torch.zeros(n + 4, device=dev)[off:off + max(n, 1)] for _ in range(4)]
        p0 = g.normal(size=n).astype(np.float32)
        bufs[0][:n].copy_(torch.from_numpy(p0))
        mask = None
        if s.get('row_len'):
            m = (g.random(n // s['row_len']) < 0.5).astype(np.uint8)
            if m.size:
                m[0], m[-1] = 0, 1
            mask = torch.from_numpy(m).to(dev)
        T.append(dict(bufs=bufs, mask=mask, dyn=torch.zeros(3, device=dev)))
        H.append([p0, np.zeros(n, np.float32), np.zeros(n, np.float32), np.zeros(n, np.float32)])
    for t in range(1, steps + 1):
        descs = []
        for s, d, h in zip(specs, T, H):
            n = s['n']
            gr = (g.normal(size=n) * s.get('gscale', 1.0)).astype(np.float32)
            if t == 3:
                gr[:] = 0
            h[1] = gr
            d['bufs'][1][:n].copy_(torch.from_numpy(gr))
            b1, b2 = s.get('betas', (0.9, 0.99))
            bc = (1.0 - b1 ** t, 1.0 - b2 ** t)
            lr = s.get('lr', 1e-2)
            dyn = None
            if s.get('dyn'):
                dyn = np.array([lr * (1 + 0.1 * t), bc[0], bc[1]], np.float32)
                d['dyn'].copy_(torch.from_numpy(dyn))
            descs.append(adam_desc(*d['bufs'], 123.0 if dyn is not None else lr, (b1, b2),
                                   s.get('eps', 1e-15), s.get('wd', 0.0),
                                   (0.5, 0.5) if dyn is not None else bc,
                                   dyn=d['dyn'].data_ptr() if dyn is not None else None,
                                   row_mask=d['mask']))
            descs[-1].n = n
            h[:] = F.adam_f32(h[0], gr, h[2], h[3], lr, b1, b2, s.get('eps', 1e-15), s.get('wd', 0.0),
                              bc[0], bc[1],
                              row_mask=None if d['mask'] is None else d['mask'].cpu().numpy(),
                              row_len=s.get('row_len') or 1, zero_grad=zero_grad,
                              dyn=None if dyn is None else tuple(dyn))
        _cabi.launch_on(dev, 'xrd_adam_step', (_cabi.XrdAdamTensor * len(descs))(*descs),
                        len(descs), zero_grad)
        torch.cuda.synchronize(dev)
        for i, (d, h) in enumerate(zip(T, H)):
            for k, name in enumerate(('param', 'grad', 'exp_avg', 'exp_avg_sq')):
                got = d['bufs'][k].cpu().numpy()[:len(h[k])]
                assert np.array_equal(_bits(got), _bits(h[k])), (t, i, name, specs[i])
    return H


ADAM_CASES = {
    'sizes': [dict(n=n) for n in (0, 1, 2, 3, 4, 5, 6, 7, 1027, 12289)],
    'misaligned': [dict(n=n, misalign=True) for n in (4, 5, 6, 7, 1027)],
    'weight_decay': [dict(n=1030, wd=1e-2, betas=(0.9, 0.999), eps=1e-8, lr=1e-3)],
    'dyn': [dict(n=1031, dyn=True), dict(n=8, dyn=True, misalign=True)],
    'mask32': [dict(n=32 * 37, row_len=32)],
    'mask3': [dict(n=3 * 41, row_len=3)],
    'mask6': [dict(n=6 * 23, row_len=6)],
    'mask32_misaligned': [dict(n=32 * 9, row_len=32, misalign=True)],
    'denormal_v': [dict(n=1024, gscale=1e-20, eps=1e-15), dict(n=7, gscale=1e-20, eps=1e-15)],
    'zero_grads': [dict(n=515, gscale=0.0)],
    'tensors25': [dict(n=5 + 13 * i) for i in range(25)],
    'tensors49': [dict(n=3 + 7 * i, misalign=bool(i % 3 == 0)) for i in range(49)],
}


@pytest.mark.gpu
@pytest.mark.parametrize('zero_grad', [0, 1])
@pytest.mark.parametrize('case', sorted(ADAM_CASES))
def test_adam_step_bit_exact(cuda_dev, case, zero_grad):
    H = _adam_steps(cuda_dev, ADAM_CASES[case], zero_grad=zero_grad)
    if case == 'denormal_v':
        v = H[0][3]
        assert ((v > 0) & (v < np.finfo(np.float32).tiny)).any()   # v really is subnormal


# ------------------------------------------------------------------ Co-SLAM sessions ---
def _jac_abs(rot, fixed):
    """|d d_rot / d G[e]| for the nine entries e of the rotation block, exactly (the backward
    is linear in G): [n, 3, 3, 3]."""
    n = rot.shape[0]
    J = np.zeros((n, 3, 3, 3))
    for e in range(9):
        G = np.zeros((n, 4, 4))
        G[:, e // 3, e % 3] = 1.0
        J[:, e // 3, e % 3] = np.abs(F.rodrigues_bwd_f64(rot, G, fixed)[0])
    return J


def _chain(rot, dirs, ids, n, d_o, d_d, fixed=None):
    """float64 d_rot / d_trans of one iteration and their bounds (the ray bound carried through
    the Rodrigues backward, plus the pose kernel's own bound with old = 0)."""
    G, A, n_p = F.rays_bwd_f64(dirs, ids, n, d_o, d_d)
    gb = F.gamma(n_p + 2)[:, None, None] * A
    d_rot, d_trans = F.rodrigues_bwd_f64(rot, G, fixed)
    b_rot = (_jac_abs(rot, fixed) * gb[:, :3, :3, None]).sum((1, 2)) + \
        _pose_bwd_bound(rot, G, d_rot)
    b_trans = gb[:, :3, 3]
    if fixed is not None:
        b_rot[np.asarray(fixed, bool)] = 0
        b_trans[np.asarray(fixed, bool)] = 0
    return d_rot, d_trans, b_rot, b_trans


@pytest.mark.gpu
def test_tracking_session_pose_chain_and_adam(cuda_dev):
    import random
    import bench
    from xrdslam_b200.coslam_graph import TrackingGraphSession
    random.seed(3)
    algo, kfs, cur = bench.build_algorithm(cuda_dev, seed=3)
    cam = algo.camera
    He, We, n = algo.config.tracking_Hedge, algo.config.tracking_Wedge, algo.config.tracking_sample
    g = torch.Generator().manual_seed(0)
    idx = torch.randint((cam.height - 2 * He) * (cam.width - 2 * We), (n,), generator=g)
    sess = TrackingGraphSession(algo, external_indices=True)
    sess.begin(cur)
    sess.idx.copy_(idx.to(cuda_dev))
    rot0, trans0 = sess.rot.cpu().numpy(), sess.trans.cpu().numpy()
    sess.step()
    torch.cuda.synchronize(cuda_dev)
    c = lambda t: t.cpu().numpy()
    d_rot, d_trans = c(sess.d_rot), c(sess.d_trans)
    ref_r, ref_t, b_r, b_t = _chain(rot0, c(sess.dirs), None, 1, c(sess.d_rays_o), c(sess.d_rays_d))
    assert np.abs(d_rot).max() > 0
    assert _note('tracking d_rot', np.abs(d_rot - ref_r), b_r) <= 1.0
    assert _note('tracking d_trans', np.abs(d_trans - ref_t), b_t) <= 1.0
    oc = algo.config.optimizers
    for name, p0, gr, got in (('tracking_pose_r', rot0, d_rot, sess.rot),
                              ('tracking_pose_t', trans0, d_trans, sess.trans)):
        o = oc[name]['optimizer']
        b1, b2 = o.betas
        dyn = np.array([o.lr, 1.0 - b1, 1.0 - b2], np.float32)   # step 1, as the ring writes them
        exp = F.adam_f32(p0, gr, np.zeros(3), np.zeros(3), 0.0, b1, b2, o.eps,
                         getattr(o, 'weight_decay', 0), 1.0, 1.0, dyn=tuple(dyn))
        assert np.array_equal(_bits(c(got).reshape(-1)), _bits(exp[0])), name


@pytest.mark.gpu
def test_mapping_session_bundle_adjustment_chain_and_adam(cuda_dev):
    import random
    import bench
    random.seed(11)
    algo, kfs, cur = bench.build_algorithm(cuda_dev, seed=11)
    algo.config.graph_mapping = True
    algo.config.min_sample_pixels = 256
    frames = kfs + [cur]
    torch.manual_seed(11)
    oc = algo.config.optimizers
    acc = oc['mapping_pose_r']['optimizer'].accum_step or 1
    algo.setup_optimizers(acc, frames, True)
    sess = algo.mapping_session(frames)
    sess.begin(frames)
    assert sess.ba and acc > 1
    c = lambda t: t.cpu().numpy()
    n = sess.n_poses
    fixed = c(sess.fixed).astype(bool)
    assert fixed[0] and not fixed.all()
    rot0, trans0 = c(sess.rot), c(sess.trans)
    sum_r, sum_t = np.zeros((n, 3)), np.zeros((n, 3))
    bnd_r, bnd_t = np.zeros((n, 3)), np.zeros((n, 3))
    prev_r, prev_t = np.zeros((n, 3), np.float32), np.zeros((n, 3), np.float32)
    for i in range(acc):
        sess.step(i, frames)
        torch.cuda.synchronize(cuda_dev)
        assert np.array_equal(c(sess.rot), rot0) or i == acc - 1
        it_r, it_t = c(sess.d_rot_it), c(sess.d_trans_it)
        ref_r, ref_t, b_r, b_t = _chain(rot0, c(sess.dirs), c(sess.ids), n, c(sess.d_rays_o),
                                        c(sess.d_rays_d), fixed)
        assert not it_r[fixed].any() and not it_t[fixed].any()
        assert _note('mapping d_rot_it', np.abs(it_r - ref_r), b_r) <= 1.0
        assert _note('mapping d_trans_it', np.abs(it_t - ref_t), b_t) <= 1.0
        sum_r, sum_t = sum_r + ref_r, sum_t + ref_t
        acc_r, acc_t = prev_r + it_r, prev_t + it_t      # the session's fp32 accumulation
        # each fp32 add rounds once: |fl(a + b) - (a + b)| <= u |fl(a + b)|
        bnd_r = bnd_r + b_r + U * np.abs(acc_r)
        bnd_t = bnd_t + b_t + U * np.abs(acc_t)
        if i < acc - 1:
            assert np.array_equal(_bits(c(sess.d_rot)), _bits(acc_r))
            assert np.array_equal(_bits(c(sess.d_trans)), _bits(acc_t))
            assert _note('mapping d_rot sum', np.abs(acc_r - sum_r), bnd_r) <= 1.0
            assert _note('mapping d_trans sum', np.abs(acc_t - sum_t), bnd_t) <= 1.0
            prev_r, prev_t = acc_r, acc_t
    # the accum_step-th iteration: one pose Adam step on the sums, zero_grad = 1
    assert not c(sess.d_rot).any() and not c(sess.d_trans).any()
    for name, p0, gr, got in (('mapping_pose_r', rot0, acc_r, sess.rot),
                              ('mapping_pose_t', trans0, acc_t, sess.trans)):
        o = oc[name]['optimizer']
        b1, b2 = o.betas
        exp = F.adam_f32(p0, gr, np.zeros(p0.size), np.zeros(p0.size), o.lr, b1, b2, o.eps,
                         getattr(o, 'weight_decay', 0), 1.0 - b1, 1.0 - b2, zero_grad=1)
        assert np.array_equal(_bits(c(got).reshape(-1)), _bits(exp[0])), name
        assert np.array_equal(c(got)[fixed], p0[fixed])


def test_report_worst(capsys):
    """Prints the worst error / bound ratio of every check run before it."""
    with capsys.disabled():
        for k in sorted(SEEN):
            print(f'  worst {k:32s} {SEEN[k]:.3g}')
