"""ds-eval depth L1 on the host: the numpy rasteriser (oracle/eval_render.py) against analytic
depth, single-triangle cases, the batched view sampler against the one-at-a-time loop,
oriented_bounds / get_cam_position on the synthetic room, and EvalMatrics' up-front check of
the unseen point cloud."""
import numpy as np
import pytest

from oracle import eval_render as ore

f32 = np.float32


def _cam(H=48, W=64, fx=50.0, fy=50.0, cx=None, cy=None, near=0.063, far=20.0):
    return dict(H=H, W=W, fx=fx, fy=fy, cx=W / 2 - 0.5 if cx is None else cx,
                cy=H / 2 - 0.5 if cy is None else cy, near=near, far=far)


def _opencv_w2c(eye, target):
    from xrdslam_b200.synthetic import look_at
    c2w = look_at(np.asarray(eye, np.float64), np.asarray(target, np.float64)).astype(np.float64)
    c2w[:3, 1:3] *= -1  # OpenGL (y up, z back) -> OpenCV (y down, z forward)
    return np.linalg.inv(c2w)[:3, :4], c2w


def _analytic(cam, c2w):
    """z-depth and hit object (0 room, 1 + k box k) of every pixel, by ray-box slabs."""
    from xrdslam_b200.synthetic import BOXES, ROOM, _slab
    j, i = np.meshgrid(np.arange(cam['H'], dtype=np.float64), np.arange(cam['W'], dtype=np.float64),
                       indexing='ij')
    d = np.stack([(i - cam['cx']) / cam['fx'], (j - cam['cy']) / cam['fy'], np.ones_like(i)], -1)
    d = d @ c2w[:3, :3].T
    o = c2w[:3, 3]
    _, t = _slab(o, d, ROOM)
    obj = np.zeros(t.shape, int)
    for k, b in enumerate(BOXES):
        tn, tf = _slab(o, d, b)
        hit = (tn < tf) & (tn > 0) & (tn < t)
        t = np.where(hit, tn, t)
        obj = np.where(hit, k + 1, obj)
    return t, obj


@pytest.mark.parametrize('eye,target', [((0.3, -0.6, 0.4), (2.0, 1.0, -1.2)),
                                        ((-0.5, -1.5, 0.9), (-2.5, -2.0, -1.0))])
def test_analytic_depth_inside_the_room(eye, target):
    from xrdslam_b200.synthetic import room_mesh
    v, f = room_mesh(0.1)
    cam = _cam()
    w2c, c2w = _opencv_w2c(eye, target)
    depth = ore.render_depth(v, f, w2c[None], cam)[0]
    t, obj = _analytic(cam, c2w)
    assert (depth > 0).all()
    pad = np.pad(obj, 1, mode='edge')
    same = np.ones(obj.shape, bool)
    for dj in (-1, 0, 1):
        for di in (-1, 0, 1):
            same &= pad[1 + dj:1 + dj + obj.shape[0], 1 + di:1 + di + obj.shape[1]] == obj
    assert same.mean() > 0.8
    assert np.abs(depth[same] - t[same]).max() < 1e-5


def _quad(z, half=0.5):
    v = np.array([[-half, -half, z], [half, -half, z], [half, half, z], [-half, half, z]], f32)
    return v, np.array([[0, 1, 2], [0, 2, 3]], np.int32)


IDENT = np.eye(4)[:3][None]


def test_fronto_parallel_quad():
    cam = _cam(fx=100.0, fy=100.0)
    v, f = _quad(2.0)
    d = ore.render_depth(v, f, IDENT, cam)[0]
    # u = 100 x / 2 + 31.5 spans [6.5, 56.5], v spans [-1.5, 48.5]: columns 7..56, every row
    cols = np.nonzero((d > 0).any(0))[0]
    assert cols.min() == 7 and cols.max() == 56 and (d[:, 7:57] == f32(2.0)).all()
    assert (d[:, :7] == 0).all() and (d[:, 57:] == 0).all()


def test_triangle_crossing_the_near_plane_is_clipped():
    cam = _cam(near=0.1)
    v = np.array([[-1.0, -0.5, 1.0], [1.0, -0.5, 1.0], [0.0, 0.8, -1.0]], f32)
    f = np.array([[0, 1, 2]], np.int32)
    d = ore.render_depth(v, f, IDENT, cam)[0]
    drawn = d > 0
    assert drawn.sum() > 50
    # the plane through the three vertices: z = 1 - 2 (y + 0.5) / 1.3 along each pixel's ray
    j, i = np.nonzero(drawn)
    dy = (j - cam['cy']) / cam['fy']
    z = (1.0 - 1.0 / 1.3) / (1.0 + 2.0 * dy / 1.3)
    assert np.abs(d[drawn] - z).max() < 1e-5 * z.max()
    assert d[drawn].min() >= f32(0.1) * (1 - 1e-6)


@pytest.mark.parametrize('z', [-2.0, 25.0])
def test_behind_the_camera_or_beyond_far_draws_nothing(z):
    cam = _cam()
    v, f = _quad(z, 3.0)
    assert (ore.render_depth(v, f, IDENT, cam) == 0).all()


def test_sliver_draws_at_most_its_line():
    cam = _cam(fx=100.0, fy=100.0)
    v = np.array([[-0.8, 0.0, 2.0], [0.8, 0.0, 2.0], [0.0, 1e-6, 2.0]], f32)
    d = ore.render_depth(v, np.array([[0, 1, 2]], np.int32), IDENT, cam)[0]
    assert (d[d > 0] == f32(2.0)).all() and (d > 0).sum() <= cam['W']


def test_depth_l1_sums_are_the_masked_sums():
    rng = np.random.default_rng(0)
    gt = rng.random((3, 37, 29)).astype(f32)
    rec = np.where(rng.random((3, 37, 29)) < 0.4, 0, rng.random((3, 37, 29))).astype(f32)
    rec[2] = 0
    s = ore.depth_l1_sums(gt, rec)
    for b in range(3):
        m = rec[b] > 0
        assert s[b, 1] == m.sum()
        assert abs(s[b, 0] - np.abs(gt[b][m] - rec[b][m]).astype(np.float64).sum()) < 1e-12


def _rigid(seed):
    from scipy.spatial.transform import Rotation
    T = np.eye(4)
    T[:3, :3] = Rotation.random(random_state=seed).as_matrix()
    T[:3, 3] = np.random.default_rng(seed).normal(size=3)
    return T


def test_oriented_bounds_recovers_the_room_box():
    from xrdslam_b200.eval_recon import oriented_bounds
    from xrdslam_b200.synthetic import ROOM, room_mesh
    v, _ = room_mesh(0.25)
    T = _rigid(3)
    vw = v.astype(np.float64) @ T[:3, :3].T + T[:3, 3]
    to_origin, ext = oriented_bounds(vw)
    size = ROOM[:, 1] - ROOM[:, 0]
    assert np.allclose(ext, np.sort(size), atol=1e-5)
    centre = T[:3, :3] @ ROOM.mean(1) + T[:3, 3]
    assert np.allclose(to_origin[:3, :3] @ centre + to_origin[:3, 3], 0, atol=1e-5)
    for row, ax in zip(to_origin[:3, :3], np.argsort(size)):
        assert abs(abs(row @ T[:3, ax]) - 1) < 1e-8
    local = vw @ to_origin[:3, :3].T + to_origin[:3, 3]
    assert (np.abs(local) <= ext / 2 + 1e-6).all()
    assert abs(np.linalg.det(to_origin[:3, :3]) - 1) < 1e-9


def test_camera_origins_lie_inside_the_room():
    from xrdslam_b200.eval_recon import get_cam_position, volume_rectangular
    from xrdslam_b200.synthetic import ROOM, room_mesh
    v, _ = room_mesh(0.25)
    ext, T = get_cam_position(v)
    o = volume_rectangular(ext, 2000, T, np.random.RandomState(0))
    assert (o > ROOM[:, 0] + 0.5).all() and (o < ROOM[:, 1] - 0.5).all()


def _unseen_patch():
    """A 2 m x 2 m patch of points on the room's +x wall."""
    a, b = np.meshgrid(np.linspace(-1.5, 0.5, 40), np.linspace(-0.5, 1.5, 40))
    return np.stack([np.full(a.size, 2.9), a.ravel(), b.ravel()], -1).astype(f32)


def test_batched_sampler_takes_the_sequential_loops_views():
    from xrdslam_b200.eval_recon import get_cam_position, sample_views
    from xrdslam_b200.synthetic import room_mesh
    v, _ = room_mesh(0.25)
    ext, T = get_cam_position(v)
    pc = _unseen_patch()
    checked = []

    def seen(c2w):
        s = np.array([ore.check_proj(pc, 500, 500, 300., 300., 249.5, 249.5, c) for c in c2w])
        checked.append(s)
        return s

    seq = ore.sample_views_sequential(pc, ext, T, 24, seed=5)
    for batch in (1, 7, 64):
        checked.clear()
        got = sample_views(pc, ext, T, 24, seed=5, batch=batch, seen_fn=seen)
        assert np.array_equal(got, seq), batch
    rejected = np.concatenate(checked).mean()
    assert 0.05 < rejected < 0.9, rejected
    with pytest.raises(RuntimeError):
        sample_views(pc, ext, T, 24, seed=5, batch=8, max_candidates=20, seen_fn=seen)


def test_eval_matrics_checks_the_unseen_cloud_first(tmp_path):
    from xrdslam_b200 import eval as ev
    from xrdslam_b200.io_formats import write_ply
    from xrdslam_b200.synthetic import room_mesh
    v, f = room_mesh(0.5)
    gt_path = write_ply(str(tmp_path / 'room.ply'), v, f)
    # no eval.tar either: the missing unseen cloud is reported before the trajectory is read
    m = ev.EvalMatrics(output_dir=tmp_path / 'missing', gt_mesh=gt_path, eval_2d_metric=True)
    with pytest.raises(ev.MissingUnseenPointCloud, match='depth renderer') as e:
        m.main()
    assert isinstance(e.value, FileNotFoundError) and isinstance(e.value, NotImplementedError)
    assert e.value.filename == str(tmp_path / 'room_pc_unseen.npy')
