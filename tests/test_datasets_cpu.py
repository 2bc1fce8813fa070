"""The dataset readers' host part (file lists, association, poses, camera), the OpenEXR depth
reader, devices.yaml inheritance, get_dataset's errors and the run CLI's --data_type / --set, on
the CPU.  Tests marked needs_reference run the reference's own classes (slam/common/datasets.py)
on the same folders."""
import os

import numpy as np
import pytest
import torch

from xrdslam_b200 import datasets as D
from xrdslam_b200 import synthetic as S

W, H = 64, 48


def _ref_module(monkeypatch):
    """The reference's datasets module; numpy 2 removed np.unicode_, which its TUM reader names."""
    from oracle import ref_harness
    ref_harness.install()
    monkeypatch.setattr(np, 'unicode_', np.str_, raising=False)
    import slam.common.datasets as R
    return R


def _assert_same_host_part(ours, ref):
    assert len(ours) == ref.n_img
    assert [os.path.basename(p) for p in ours.color_paths] == \
        [os.path.basename(p) for p in ref.color_paths]
    assert [os.path.basename(p) for p in ours.depth_paths] == \
        [os.path.basename(p) for p in ref.depth_paths]
    assert [os.path.normpath(p) for p in ours.color_paths] == \
        [os.path.normpath(p) for p in ref.color_paths]
    assert len(ours.poses) == len(ref.poses)
    for a, b in zip(ours.poses, ref.poses):
        assert a.dtype == b.dtype == torch.float32
        assert np.array_equal(a.numpy().view(np.int32), b.numpy().view(np.int32))
    c, r = ours.camera, ref.camera
    assert (c.fx, c.fy, c.cx, c.cy, c.height, c.width) == (r.fx, r.fy, r.cx, r.cy, r.height,
                                                           r.width)
    assert ours.png_depth_scale == ref.png_depth_scale
    assert ours.crop_edge == ref.crop_edge and ours.downsample_factor == ref.downsample_factor
    assert (ours.distortion is None) == (ref.distortion is None)
    if ours.distortion is not None:
        assert np.array_equal(ours.distortion, ref.distortion)


DIST5 = [0.2624, -0.9531, -0.0054, 0.0026, 1.1633]
# key, reference class, writer, writer keywords
LAYOUTS = [
    ('tumrgbd', 'TUM_RGBD', S.write_tum, dict(n_frames=6)),
    ('tumrgbd', 'TUM_RGBD', S.write_tum, dict(n_frames=4, distortion=DIST5, crop_edge=3,
                                              downsample_factor=2, seed=3)),
    ('scannet', 'ScanNet', S.write_scannet, dict(n_frames=12, crop_edge=2)),
    ('7scenes', 'Scenes7', S.write_7scenes, dict(n_frames=3)),
    ('azure', 'Azure', S.write_azure, dict(n_frames=3)),
    ('azure', 'Azure', S.write_azure, dict(n_frames=3, trajectory_log=False)),
    ('cofusion', 'CoFusion', S.write_cofusion, dict(n_frames=3, downsample_factor=2)),
]


@pytest.fixture(scope='module')
def layouts(tmp_path_factory):
    out = []
    for k, (key, _, writer, kw) in enumerate(LAYOUTS):
        folder = str(tmp_path_factory.mktemp(f'{key}{k}'))
        writer(folder, width=W, height=H, **kw)
        out.append(folder)
    return out


@pytest.mark.parametrize('case', range(len(LAYOUTS)))
def test_synthetic_layout_reads_back(layouts, case):
    key, _, writer, kw = LAYOUTS[case]
    ds = D.get_dataset(layouts[case], key, device='cpu')
    n = kw['n_frames']
    assert len(ds) == n == len(ds.depth_paths)
    cam = S.make_camera(W, H)
    e, f = kw.get('crop_edge', 0), kw.get('downsample_factor', 1)
    assert (ds.camera.height, ds.camera.width) == (int((H - 2 * e) / f), int((W - 2 * e) / f))
    assert ds.fx == cam.fx and ds.cy == cam.cy
    gt = S.trajectory(n)
    for k in range(n):
        if key == 'cofusion' or kw.get('trajectory_log') is False:
            assert torch.equal(ds.poses[k], torch.eye(4))
        else:  # the written float64 pose, flipped back (TUM through its quaternion)
            assert np.allclose(ds.poses[k].numpy(), gt[k], atol=1e-6)
    color, depth = ds.read_raw(0)
    assert color.dtype == torch.uint8 and color.shape[-1] == 3
    assert depth.dtype == (torch.float32 if key == 'cofusion' else torch.int16)
    if key in ('scannet', 'azure'):  # colour larger than depth: the ingest resizes it
        assert color.shape[:2] != depth.shape
    if key == 'cofusion':
        d = depth.numpy()
        assert np.isnan(d).any() and (d == 0).any()


@pytest.mark.needs_reference
@pytest.mark.parametrize('case', range(len(LAYOUTS)))
def test_reader_equals_reference(layouts, monkeypatch, case):
    key, cls, _, _ = LAYOUTS[case]
    R = _ref_module(monkeypatch)
    _assert_same_host_part(D.get_dataset(layouts[case], key, device='cpu'),
                           getattr(R, cls)(layouts[case], device='cpu'))


# ---- TUM RGB-D edge cases -------------------------------------------------------------------
def _tum_folder(root, rgb_t, depth_t, pose_rows, pose_name='groundtruth.txt', header=True):
    os.makedirs(root, exist_ok=True)
    with open(os.path.join(root, 'devices.yaml'), 'w') as f:
        f.write('cam:\n  H: 480\n  W: 640\n  fx: 517.3\n  fy: 516.5\n  cx: 318.6\n  cy: 255.3\n'
                '  png_depth_scale: 5000.0\n  crop_edge: 8\n'
                '  distortion: [0.2624, -0.9531, -0.0054, 0.0026, 1.1633]\n')
    for name, ts in (('rgb', rgb_t), ('depth', depth_t)):
        with open(os.path.join(root, f'{name}.txt'), 'w') as f:
            f.write('# color images\n# file: x\n# timestamp filename\n')
            for t in ts:
                f.write(f'{t:.6f} {name}/{t:.6f}.png\n')
    with open(os.path.join(root, pose_name), 'w') as f:
        if header:
            f.write('# ground truth trajectory\n# file: x\n# timestamp tx ty tz qx qy qz qw\n')
        for row in pose_rows:
            f.write(' '.join(f'{v:.17g}' if i else f'{v:.4f}' for i, v in enumerate(row)) + '\n')
    return root


def _pose_rows(ts, seed):
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(seed)
    q = Rotation.random(len(ts), random_state=seed).as_quat()
    return [[t, *rng.normal(size=3), *qq] for t, qq in zip(ts, q)]


def _tum_expected(rows, keep):
    """float32 c2w of the pose rows `keep`, built as the reference builds them."""
    from scipy.spatial.transform import Rotation
    out = []
    for k in keep:
        p = np.eye(4)
        v = np.array(rows[k][1:], np.float64)
        p[:3, :3] = Rotation.from_quat(v[3:]).as_matrix()
        p[:3, 3] = v[:3]
        p[:3, 1] *= -1
        p[:3, 2] *= -1
        out.append(torch.from_numpy(p).float())
    return out


def _tum_cases(tmp_path):
    t0 = 1311868164.0
    # images: 0, 0.02 (< 1/32 s after 0: dropped), 0.1, 0.2 (nearest depth 0.1 away: dropped),
    # 0.3 (nearest pose 0.1 away: dropped), 0.4, 0.41 (dropped), 0.45 (kept: 0.05 after 0.4)
    rgb = [t0 + d for d in (0.0, 0.02, 0.1, 0.2, 0.3, 0.4, 0.41, 0.45)]
    dep = [t0 + d for d in (0.003, 0.021, 0.098, 0.31, 0.402, 0.412, 0.449)]
    pose_t = [t0 + d for d in (0.001, 0.099, 0.2, 0.399, 0.45)]
    rows = _pose_rows(pose_t, 0)
    yield 'groundtruth', _tum_folder(str(tmp_path / 'gt'), rgb, dep, rows), \
        [0, 2, 5, 7], [0, 1, 3, 4], rows
    # a pose.txt without a header loses its first row to skiprows=1: image 0 has no pose within
    # 0.08 s any more and is dropped, image 1 (0.079 s from the second pose) is kept in its place
    rows2 = _pose_rows(pose_t, 1)
    yield 'headerless pose.txt', _tum_folder(str(tmp_path / 'pose'), rgb, dep, rows2,
                                             pose_name='pose.txt', header=False), \
        [1, 2, 5, 7], [1, 1, 3, 4], rows2


def test_tum_association_subsampling_and_headerless_pose(tmp_path):
    for name, folder, keep_img, keep_pose, rows in _tum_cases(tmp_path):
        ds = D.TUM_RGBD(folder, device='cpu')
        rgb = D.tum_parse_list(os.path.join(folder, 'rgb.txt'))
        assert [os.path.basename(p) for p in ds.color_paths] == \
            [os.path.basename(rgb[i, 1]) for i in keep_img], name
        exp = _tum_expected(rows, keep_pose)
        assert len(ds.poses) == len(exp)
        for a, b in zip(ds.poses, exp):
            assert torch.equal(a, b), name
        assert ds.camera.width == 640 - 16 and np.array_equal(ds.distortion, DIST5)


@pytest.mark.needs_reference
def test_tum_edge_cases_equal_reference(tmp_path, monkeypatch):
    R = _ref_module(monkeypatch)
    for name, folder, _, _, _ in _tum_cases(tmp_path):
        _assert_same_host_part(D.TUM_RGBD(folder, device='cpu'), R.TUM_RGBD(folder, device='cpu'))


def test_tum_without_pose_file_names_both(tmp_path):
    folder = _tum_folder(str(tmp_path), [1.0], [1.0], [[1.0, 0, 0, 0, 0, 0, 0, 1]])
    os.remove(os.path.join(folder, 'groundtruth.txt'))
    with pytest.raises(FileNotFoundError, match='groundtruth.txt.*pose.txt'):
        D.TUM_RGBD(folder, device='cpu')


# ---- ScanNet, 7-Scenes and Azure edge cases ------------------------------------------------
def _devices(root, extra=''):
    with open(os.path.join(root, 'devices.yaml'), 'w') as f:
        f.write('cam:\n  H: 480\n  W: 640\n  fx: 577.59\n  fy: 578.73\n  cx: 318.9\n  cy: 242.68\n'
                f'  png_depth_scale: 1000.0\n{extra}')


def _scannet_numeric(tmp_path):
    root = tmp_path / 'scannet'
    fr = root / 'frames'
    for sub in ('color', 'depth', 'pose'):
        (fr / sub).mkdir(parents=True)
    rng = np.random.default_rng(5)
    mats = {}
    for k in (10, 9, 0, 11, 1, 2, 100):  # '10' < '9' and '100' < '11' lexicographically
        (fr / 'color' / f'{k}.jpg').write_bytes(b'')
        (fr / 'depth' / f'{k}.png').write_bytes(b'')
        m = rng.normal(size=(4, 4))
        if k == 2:
            m[:] = -np.inf  # ScanNet marks lost frames this way
        mats[k] = m
        with open(fr / 'pose' / f'{k}.txt', 'w') as f:
            for row in m:
                f.write(' '.join(repr(float(v)) for v in row) + '\n')
    _devices(str(root), '  crop_edge: 10\n')
    return str(root), mats


def test_scannet_sorts_by_frame_number(tmp_path):
    root, mats = _scannet_numeric(tmp_path)
    ds = D.ScanNet(root, device='cpu')
    order = [0, 1, 2, 9, 10, 11, 100]
    assert [os.path.basename(p) for p in ds.color_paths] == [f'{k}.jpg' for k in order]
    assert [os.path.basename(p) for p in ds.depth_paths] == [f'{k}.png' for k in order]
    for k, p in zip(order, ds.poses):
        m = mats[k].copy()
        m[:3, 1] *= -1
        m[:3, 2] *= -1
        assert torch.equal(p, torch.from_numpy(m).float())
    assert torch.isinf(ds.poses[2]).all()


@pytest.mark.needs_reference
def test_scannet_numeric_order_equals_reference(tmp_path, monkeypatch):
    R = _ref_module(monkeypatch)
    root, _ = _scannet_numeric(tmp_path)
    ours, ref = D.ScanNet(root, device='cpu'), R.ScanNet(root, device='cpu')
    assert len(ours) == ref.n_img
    assert ours.color_paths == ref.color_paths and ours.depth_paths == ref.depth_paths
    for a, b in zip(ours.poses, ref.poses):
        assert np.array_equal(a.numpy(), b.numpy(), equal_nan=True)


def test_7scenes_sorts_by_number_after_the_last_dash(tmp_path):
    root = tmp_path / 's7'
    root.mkdir()
    for k in (12, 3, 100):
        for kind in ('color.png', 'depth.png'):
            (root / f'frame-{k:d}.{kind}').write_bytes(b'')
        with open(root / f'frame-{k:d}.pose.txt', 'w') as f:
            for r in range(4):
                f.write('\t'.join(str(float(k + r + c)) for c in range(4)) + '\t\n')
    _devices(str(root))
    ds = D.Scenes7(str(root), device='cpu')
    assert [os.path.basename(p) for p in ds.color_paths] == \
        ['frame-3.color.png', 'frame-12.color.png', 'frame-100.color.png']
    assert float(ds.poses[1][0, 0]) == 12.0 and float(ds.poses[2][0, 1]) == -101.0


def test_azure_trajectory_log_blocks(tmp_path):
    folder = str(tmp_path / 'az')
    S.write_azure(folder, 2, width=W, height=H)
    ds = D.Azure(folder, device='cpu')
    gt = S.trajectory(2)
    assert len(ds.poses) == 2 and all(np.allclose(p.numpy(), g, atol=1e-7)
                                      for p, g in zip(ds.poses, gt))
    os.remove(os.path.join(folder, 'scene', 'trajectory.log'))
    ds = D.Azure(folder, device='cpu')
    assert len(ds.poses) == 2 and all(torch.equal(p, torch.eye(4)) for p in ds.poses)


# ---- OpenEXR depth --------------------------------------------------------------------------
def _special_f32(shape, seed):
    rng = np.random.default_rng(seed)
    d = rng.uniform(-2.0, 8.0, shape).astype(np.float32)
    flat = d.reshape(-1)
    specials = np.array([np.nan, np.inf, -np.inf, 0.0, -0.0, -1.5, 1e-40, -3e-42, 1e-45,
                         3e38, -3e38, 65535.0], np.float32)
    idx = rng.choice(flat.size, size=flat.size // 4, replace=False)
    flat[idx] = specials[rng.integers(0, specials.size, idx.size)]
    flat.view(np.uint32)[idx[:7]] = [0x7fc12345, 0xffc00001, 0x7fa00000, 0x7f800001, 0x7fffffff,
                                     0xff800001, 0x7fc00000]  # NaN payloads, signalling ones too
    return d


def test_exr_reader_keeps_every_bit(tmp_path):
    cv2 = pytest.importorskip('cv2')
    d = _special_f32((37, 53), 0)
    os.environ.setdefault('OPENCV_IO_ENABLE_OPENEXR', '1')
    path = str(tmp_path / 'depth.exr')
    assert cv2.imwrite(path, d)
    got = D.read_depth_exr(path)
    assert got.dtype == np.float32 and got.shape == d.shape
    # OpenEXR stores what cv2 hands it: compare with cv2's own decode, and with the array
    ref = cv2.imread(path, cv2.IMREAD_UNCHANGED)
    assert np.array_equal(got.view(np.uint32), ref.view(np.uint32))
    finite = ~np.isnan(d)
    assert np.array_equal(got.view(np.uint32)[finite], d.view(np.uint32)[finite])
    assert np.array_equal(np.isnan(got), np.isnan(d))
    assert D.read_depth_any(path).dtype == np.float32


def test_exr_reader_rejects_what_it_cannot_use(tmp_path):
    cv2 = pytest.importorskip('cv2')
    os.environ.setdefault('OPENCV_IO_ENABLE_OPENEXR', '1')
    path = str(tmp_path / 'rgb.exr')
    assert cv2.imwrite(path, np.ones((4, 5, 3), np.float32))
    with pytest.raises(ValueError, match='single-channel'):
        D.read_depth_exr(path)
    with pytest.raises(FileNotFoundError):
        D.read_depth_exr(str(tmp_path / 'missing.exr'))
    bad = tmp_path / 'bad.exr'
    bad.write_bytes(b'not an exr file')
    with pytest.raises((RuntimeError, ValueError)):
        D.read_depth_exr(str(bad))
    with pytest.raises(ValueError, match='.png or an .exr'):
        D.read_depth_any(str(tmp_path / 'depth.tiff'))


# ---- the float-depth oracle against the reference's __getitem__ -----------------------------
@pytest.mark.needs_reference
@pytest.mark.parametrize('edge,f', [(0, 1), (3, 1), (0, 2), (3, 3)])
def test_float_depth_oracle_equals_reference_getitem(tmp_path, monkeypatch, edge, f):
    from ingest_f32_oracle import ingest_f32
    R = _ref_module(monkeypatch)
    folder = str(tmp_path / 'cof')
    S.write_cofusion(folder, 2, width=W, height=H, crop_edge=edge, downsample_factor=f)
    arrays = [_special_f32((H, W), 10 + k) for k in range(2)]
    monkeypatch.setattr(R, 'readEXR_onlydepth',
                        lambda p: arrays[int(os.path.basename(p)[5:9])].copy())
    ref = R.CoFusion(folder, device='cpu')
    ours = D.CoFusion(folder, device='cpu')
    for k in range(2):
        _, rgb_r, dep_r, _ = ref[k]
        color, _ = ours.read_raw(k)
        rgb_o, dep_o = ingest_f32(color.numpy(), arrays[k], ours.fx, ours.fy, ours.cx, ours.cy,
                                  ours.distortion, ours.png_depth_scale, edge, f)
        assert np.array_equal(dep_r.numpy().view(np.uint32), dep_o.view(np.uint32))
        if f == 1:  # copies: bit for bit
            assert np.array_equal(rgb_r.numpy().view(np.uint32), rgb_o.view(np.uint32))
        else:  # INTER_LINEAR of f64 colour: cv2 with IPP differs by up to ~2e-6
            assert np.abs(rgb_r.numpy() - rgb_o).max() < 2e-6


def test_float_depth_oracle_divides_as_numpy():
    from ingest_f32_oracle import ingest_f32
    d = _special_f32((20, 30), 7)
    c = np.zeros((20, 30, 3), np.uint8)
    _, dep = ingest_f32(c, d, 10., 10., 15., 10., None, 5000.0, 2, 2)
    with np.errstate(invalid='ignore', under='ignore'):
        exp = (d / np.float32(5000.0))[2:-2, 2:-2][0::2, 0::2]
    assert np.array_equal(dep.view(np.uint32), exp.view(np.uint32))


# ---- devices.yaml inheritance, get_dataset ---------------------------------------------------
def _inherit_files(tmp_path):
    base = tmp_path / 'configs'
    base.mkdir()
    (base / 'tum.yaml').write_text('cam:\n  H: 480\n  W: 640\n  png_depth_scale: 5000.0\n'
                                   '  crop_edge: 8\n  fx: 1.0\n  fy: 1.0\n  cx: 1.0\n  cy: 1.0\n'
                                   'mapping:\n  bound: [[0, 1], [0, 1], [0, 1]]\n')
    scene = tmp_path / 'scene'
    scene.mkdir()
    (scene / 'devices.yaml').write_text('inherit_from: ../configs/tum.yaml\ncam:\n  fx: 517.3\n'
                                        '  fy: 516.5\n  cx: 318.6\n  cy: 255.3\n')
    return str(scene / 'devices.yaml')


def test_load_config_inherits_recursively(tmp_path):
    cfg = D.load_config(_inherit_files(tmp_path))
    assert cfg['cam'] == dict(H=480, W=640, png_depth_scale=5000.0, crop_edge=8, fx=517.3,
                              fy=516.5, cx=318.6, cy=255.3)
    assert cfg['mapping']['bound'] == [[0, 1], [0, 1], [0, 1]]
    assert cfg['inherit_from'] == '../configs/tum.yaml'


@pytest.mark.needs_reference
def test_load_config_equals_reference(tmp_path, monkeypatch):
    _ref_module(monkeypatch)
    from slam.utils.config import load_config
    path = _inherit_files(tmp_path)
    monkeypatch.chdir(os.path.dirname(path))  # the reference resolves inherit_from from here
    assert D.load_config(path) == load_config(path)


def test_get_dataset_errors():
    with pytest.raises(NotImplementedError, match='MonoImu'):
        D.get_dataset('/nonexistent', 'euroc')
    with pytest.raises(ValueError) as e:
        D.get_dataset('/nonexistent', 'kitti')
    for key in ('replica', 'tumrgbd', 'scannet', '7scenes', 'azure', 'cofusion'):
        assert repr(key) in str(e.value)
    assert sorted(D.dataset_dict) == sorted(['replica', 'tumrgbd', 'scannet', '7scenes', 'azure',
                                             'cofusion'])


def test_frame_ingest_rejects_other_depth_types():
    c = torch.zeros(1, 4, 4, 3, dtype=torch.uint8)
    for dt in (torch.float64, torch.int32, torch.uint8, torch.float16):
        with pytest.raises(TypeError):
            D.frame_ingest(c, torch.zeros(1, 4, 4, dtype=dt), 1., 1., 1., 1.)


# ---- the CLI: --data_type and --set ---------------------------------------------------------
def test_cli_data_type_choices():
    from xrdslam_b200 import run
    ap = run.parser()
    action = next(a for a in ap._actions if a.dest == 'data_type')
    assert sorted(action.choices) == sorted(D.dataset_dict) and action.default == 'replica'
    assert ap.parse_args(['co-slam', '--data', 'x']).data_type == 'replica'
    assert ap.parse_args(['co-slam', '--data', 'x', '--data-type', 'tumrgbd']).data_type == \
        'tumrgbd'
    with pytest.raises(SystemExit):
        ap.parse_args(['co-slam', '--data', 'x', '--data_type', 'euroc'])


def test_parse_set():
    from xrdslam_b200.run import parse_set
    got = parse_set(['mapping_bound=[[-1, 1], [-2, 2.5], [0, 3]]', 'tracking_n_iters=7',
                     'mesher.resolution = 128', 'keyframe_selection_method=all',
                     'tracker.use_relative_pose=True', 'tracking_n_iters=8', 'x=-1e-3'])
    assert got == {'mapping_bound': [[-1, 1], [-2, 2.5], [0, 3]], 'tracking_n_iters': 8,
                   'mesher.resolution': 128, 'keyframe_selection_method': 'all',
                   'tracker.use_relative_pose': True, 'x': -1e-3}
    for bad in ('tracking_n_iters', '=3'):
        with pytest.raises(ValueError):
            parse_set([bad])


def test_set_reaches_every_config():
    from xrdslam_b200 import pipeline as P
    from xrdslam_b200.run import parse_set
    bound = [[-3.2, 3.2], [-4.2, 2.7], [-2.2, 2.7]]
    cfg = P.make_config('co-slam', **parse_set([
        f'mapping_bound={bound}', 'tracking_n_iters=3', 'model.cam_depth_trunc=5.0',
        'mesher.resolution=64', 'tracker.render_freq=5', 'mapper.keyframe_every=2']))
    assert cfg.algorithm.mapping_bound == bound and cfg.algorithm.tracking_n_iters == 3
    assert cfg.algorithm.model.cam_depth_trunc == 5.0 and cfg.algorithm.mesher.resolution == 64
    assert cfg.tracker.render_freq == 5 and cfg.mapper.keyframe_every == 2
    # the preset's other values stay
    ref = P.make_config('co-slam')
    assert cfg.tracker.map_every == ref.tracker.map_every == 5
    assert cfg.algorithm.mesher.points_batch_size == ref.algorithm.mesher.points_batch_size
    assert cfg.algorithm.model.tcnn_encoding == ref.algorithm.model.tcnn_encoding
    for bad in ('no_such_field', 'model.no_such_field', 'tracker.no_such', 'decoder.x',
                'model.x.y'):
        with pytest.raises(ValueError):
            P.make_config('co-slam', **{bad: 1})
    with pytest.raises(ValueError):  # Vox-Fusion's config has no mesher
        P.make_config('vox-fusion', **{'mesher.resolution': 64})


def test_cli_unknown_field_fails_before_any_work(tmp_path, monkeypatch):
    from xrdslam_b200 import pipeline as P
    from xrdslam_b200 import run

    def no_run(*a, **k):
        raise AssertionError('the run started')
    monkeypatch.setattr(P, 'XRDSLAM', no_run)
    for sets in (['no_such_field=1'], ['mapper.nope=2'], ['tracking_n_iters']):
        with pytest.raises(SystemExit) as e:
            run.main(['co-slam', '--data', str(tmp_path / 'missing'), '--data_type', 'tumrgbd',
                      *sum((['--set', s] for s in sets), [])])
        assert e.value.code == 2
