"""TSDF fusion, coloured marching cubes and clean_mesh on the device (csrc/tsdf.cu,
xrdslam_b200/tsdf.py) bit for bit against the numpy restatement (oracle/tsdf.py), and
PointSLAM.get_mesh end to end."""
import numpy as np
import pytest
import torch

from oracle import tsdf as ot

pytestmark = pytest.mark.gpu
f32 = np.float32


def _seq(n, width=160, height=120, offset=(0.0, 0.0, 0.0)):
    from xrdslam_b200.synthetic import make_sequence
    cam, poses, frames = make_sequence(n, width=width, height=height, offset=offset)
    c2w, w2c = ot.o3d_poses(poses)
    depth = np.stack([d for _, d in frames])
    color = np.stack([(rgb * 255).astype(np.uint8) for rgb, _ in frames])
    return cam, poses, depth, color, c2w, w2c


def _intr(cam):
    return (cam.fx, cam.fy, cam.cx, cam.cy)


def _bits(a):
    a = a.detach().cpu().numpy() if torch.is_tensor(a) else np.asarray(a)
    return a.view(np.uint32) if a.dtype == np.float32 else a


def _assert_eq(a, b):
    a, b = _bits(a), _bits(b)
    assert a.shape == b.shape, (a.shape, b.shape)
    assert np.array_equal(a, b)


def _fuse(dev, depth, color, c2w, w2c, intr, batches=None):
    """Device volume and oracle volume from the same frames (optionally in several batches)."""
    from xrdslam_b200.tsdf import TSDFVolume
    vol = TSDFVolume(device=dev)
    ora = ot.Volume(ot.Params(intr))
    batches = batches or [slice(0, depth.shape[0])]
    for s in batches:
        vol.integrate(torch.from_numpy(depth[s]).to(dev), torch.from_numpy(color[s]).to(dev),
                      c2w[s], intr, w2c=w2c[s])
        ora.integrate(depth[s], color[s], c2w[s], w2c[s])
    torch.cuda.synchronize()
    return vol, ora


def _check_volume(vol, ora):
    _assert_eq(vol.keys, ora.keys)
    _assert_eq(vol.tsdf, ora.tsdf)
    _assert_eq(vol.weight, ora.weight)
    _assert_eq(vol.color, ora.color)


def _check_mesh(vol, ora, min_faces=1):
    from xrdslam_b200.tsdf import clean_mesh_arrays
    v, f, c = vol.extract_triangle_mesh()
    ov, of, oc = ora.extract()
    _assert_eq(v, ov)
    _assert_eq(f, of)
    _assert_eq(c, oc)
    assert of.shape[0] >= min_faces
    cv, cf, cc = clean_mesh_arrays(v, f, c)
    ocv, ocf, occ = ot.clean_mesh(ov, of, oc)
    _assert_eq(cv, ocv)
    _assert_eq(cf, ocf)
    _assert_eq(cc, occ)
    return ov, of, oc


def test_allocation_masks_and_volume_160x120(cuda_dev):
    cam, _, depth, color, c2w, w2c = _seq(3)
    from xrdslam_b200.tsdf import TSDFVolume
    vol = TSDFVolume(device=cuda_dev)
    keys, masks = vol.allocate(torch.from_numpy(depth).to(cuda_dev),
                               torch.from_numpy(c2w[:, :3].copy()).to(cuda_dev), _intr(cam))
    okeys, omasks = ot.allocate(depth, c2w, ot.Params(cam))
    _assert_eq(keys, okeys)
    _assert_eq(masks.cpu().numpy().view(np.uint32), omasks)
    vol, ora = _fuse(cuda_dev, depth, color, c2w, w2c, _intr(cam))
    _check_volume(vol, ora)
    assert (ora.weight == 3).sum() > 10000
    _check_mesh(vol, ora, min_faces=5000)


def test_full_size_640x480(cuda_dev):
    cam, _, depth, color, c2w, w2c = _seq(2, 640, 480)
    vol, ora = _fuse(cuda_dev, depth, color, c2w, w2c, _intr(cam))
    assert vol.n_blocks > 5000
    _check_volume(vol, ora)
    _check_mesh(vol, ora, min_faces=100000)


def test_single_frame(cuda_dev):
    cam, _, depth, color, c2w, w2c = _seq(1)
    vol, ora = _fuse(cuda_dev, depth, color, c2w, w2c, _intr(cam))
    assert set(np.unique(ora.weight)) == {0, 1}
    _check_volume(vol, ora)
    _check_mesh(vol, ora, min_faces=1000)


def test_more_than_32_keyframes_cross_a_mask_word(cuda_dev):
    cam, _, depth, color, c2w, w2c = _seq(37, 64, 48)
    vol, ora = _fuse(cuda_dev, depth, color, c2w, w2c, _intr(cam))
    _, omasks = ot.allocate(depth, c2w, ot.Params(cam))
    assert omasks.shape[1] == 2
    assert ((omasks[:, 0] != 0) & (omasks[:, 1] != 0)).sum() > 10   # blocks of both words
    _check_volume(vol, ora)
    _check_mesh(vol, ora, min_faces=1000)


def test_negative_world_coordinates(cuda_dev):
    cam, _, depth, color, c2w, w2c = _seq(2, offset=(-40.0, -25.5, -13.0))
    vol, ora = _fuse(cuda_dev, depth, color, c2w, w2c, _intr(cam))
    assert (ot.unpack(ora.keys) < 0).all()
    _check_volume(vol, ora)
    _check_mesh(vol, ora, min_faces=5000)


def test_voxels_on_the_last_image_row_and_column(cuda_dev):
    # depth only on the last row and column (both sampled: H - 1 and W - 1 are multiples of 4):
    # every updated voxel projected there
    H, W = 41, 61
    intr = (40.0, 40.0, 30.0, 20.0)
    depth = np.zeros((1, H, W), f32)
    depth[0, H - 1, :] = 1.5
    depth[0, :, W - 1] = 1.7
    color = np.random.default_rng(0).integers(0, 256, (1, H, W, 3)).astype(np.uint8)
    c2w = np.eye(4, dtype=f32)[None].copy()
    w2c = c2w.copy()
    vol, ora = _fuse(cuda_dev, depth, color, c2w, w2c, intr)
    assert (ora.weight > 0).sum() > 1000
    _check_volume(vol, ora)


def test_mesh_ends_at_unallocated_neighbour_blocks(cuda_dev):
    # a small tilted plane patch: its blocks border unallocated ones on every side
    H, W = 64, 64
    intr = (60.0, 60.0, 31.5, 31.5)
    v, u = np.mgrid[0:H, 0:W].astype(np.float64)
    depth = (1.0 + 0.004 * u + 0.002 * v).astype(f32)[None]
    color = np.full((1, H, W, 3), 128, np.uint8)
    c2w = np.eye(4, dtype=f32)[None].copy()
    vol, ora = _fuse(cuda_dev, depth, color, c2w, c2w.copy(), intr)
    nbr = ot.neighbours(ora.keys)
    assert (nbr[:, 1:] < 0).any()
    ov, of, _ = _check_mesh(vol, ora, min_faces=500)
    # no face reaches across a missing block: every edge is shorter than a cube diagonal
    e = np.linalg.norm(ov[of] - ov[np.roll(of, 1, 1)], axis=2)
    assert e.max() <= np.sqrt(3) * 4 / 512 + 1e-6
    assert of.max() < ov.shape[0]


def test_clean_mesh_components_of_99_and_100_vertices(cuda_dev):
    from test_tsdf_cpu import _strip
    from xrdslam_b200.tsdf import clean_mesh_arrays, components
    v99, f99 = _strip(99, 0.0)
    v100, f100 = _strip(100, 1000.0)
    v = np.concatenate([v99, v100, v100[:1]])
    f = np.concatenate([f99, f100 + 99, f100[:1] + 99, [[99, 100, 199]]]).astype(np.int32)
    c = np.random.default_rng(0).random(v.shape, dtype=f32)
    lab = components(torch.from_numpy(f).to(cuda_dev), v.shape[0])
    _assert_eq(lab.cpu().numpy().astype(np.int64), ot.components(f, v.shape[0]))
    cv, cf, cc = clean_mesh_arrays(*(torch.from_numpy(a).to(cuda_dev) for a in (v, f, c)))
    ocv, ocf, occ = ot.clean_mesh(v, f, c)
    assert ocv.shape[0] == 100
    _assert_eq(cv, ocv)
    _assert_eq(cf, ocf)
    _assert_eq(cc, occ)


def test_storage_grows_across_two_integrate_calls(cuda_dev):
    cam, _, depth, color, c2w, w2c = _seq(4)
    from xrdslam_b200.tsdf import TSDFVolume
    vol, ora = _fuse(cuda_dev, depth, color, c2w, w2c, _intr(cam), [slice(0, 2), slice(2, 4)])
    first = TSDFVolume(device=cuda_dev)
    first.integrate(torch.from_numpy(depth[:2]).to(cuda_dev), torch.from_numpy(color[:2]).to(cuda_dev),
                    c2w[:2], _intr(cam), w2c=w2c[:2])
    assert vol.n_blocks > first.n_blocks
    _check_volume(vol, ora)
    one, _ = _fuse(cuda_dev, depth, color, c2w, w2c, _intr(cam))
    for a in ('keys', 'tsdf', 'weight', 'color'):
        _assert_eq(getattr(vol, a), getattr(one, a))
    _check_mesh(vol, ora, min_faces=5000)


# ---- PointSLAM.get_mesh ------------------------------------------------------------------------
def _point_slam(dev, n_frames=2, clean=True):
    from test_algorithms_gpu import _frames, _losses
    from xrdslam_b200.point_slam import PointSLAMConfig
    torch.manual_seed(0)
    np.random.seed(0)
    cam, poses, fr = _frames(n_frames, separate_LR=True)
    cfg = PointSLAMConfig(pixels_adding=1500, mapping_sample=1000, tracking_sample=300,
                          tracking_Wedge=10, tracking_Hedge=10, clean_mesh=clean)
    algo = cfg.setup(camera=cam, device=dev)
    return algo, cam, fr, _losses


def _oracle_mesh(cam, keyframes, clean):
    c2w, w2c = ot.o3d_poses([kf.get_pose().detach().cpu().numpy() for kf in keyframes])
    depth = np.stack([np.asarray(kf.depth, f32) for kf in keyframes])
    color = np.stack([(np.asarray(kf.rgb, f32) * f32(255)).astype(np.uint8) for kf in keyframes])
    ora = ot.Volume(ot.Params(cam))
    ora.integrate(depth, color, c2w, w2c)
    v, f, c = ora.extract()
    v = v + np.array([-0.0 / 512.0, 2.5 / 512.0, -2.5 / 512.0], f32)
    if clean:
        v, f, c = ot.clean_mesh(v, f, c)
        return v, f, ot.colors_to_u8(c)
    return v, f, None


@pytest.mark.parametrize('clean', [True, False])
def test_point_slam_get_mesh_end_to_end(cuda_dev, tmp_path, clean):
    from xrdslam_b200 import io_formats
    algo, cam, fr, losses = _point_slam(cuda_dev, clean=clean)
    assert algo.get_mesh() is None                      # no keyframe yet
    for k in range(2):
        algo.add_keyframe(fr[k])
        losses(algo, [fr[k]], 6, True)
        algo.set_initialized()
    mesh = algo.get_mesh()
    assert mesh is not None and mesh.faces.shape[0] > 1000
    ov, of, oc = _oracle_mesh(cam, algo.keyframe_graph, clean)
    _assert_eq(mesh.vertices, ov)
    _assert_eq(mesh.faces, of)
    if clean:
        assert mesh.vertex_colors.dtype == np.uint8
        _assert_eq(mesh.vertex_colors, oc)
    else:
        assert mesh.vertex_colors is None
    p = mesh.export(str(tmp_path / 'final_mesh.ply'))
    v2, f2, c2 = io_formats.read_ply(p)
    assert np.array_equal(v2, mesh.vertices) and np.array_equal(f2, mesh.faces)
    if clean:
        assert np.array_equal(c2, mesh.vertex_colors)


def test_point_slam_get_mesh_all_zero_depth_is_none(cuda_dev):
    from xrdslam_b200.frame import Frame
    algo, cam, fr, _ = _point_slam(cuda_dev, n_frames=1)
    f0 = fr[0]
    blank = Frame(0, f0.rgb, np.zeros_like(f0.depth), init_pose=f0.get_pose().detach().cpu().numpy(),
                  separate_LR=True, rot_rep='axis_angle')
    algo.add_keyframe(blank)
    assert algo.get_mesh() is None
