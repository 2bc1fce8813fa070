"""The run's control flow, pose prediction, presets and the Replica reader's host part, on the CPU:
a recording fake Algorithm driven by XRDSLAM.run() against a restatement of the reference's
tracker.spin / mapper.spin (slam/pipeline/tracker.py:52-183, mapper.py:20-46)."""
import ast
import os

import numpy as np
import pytest
import torch

from xrdslam_b200 import pipeline as P
from xrdslam_b200.camera import Camera
from xrdslam_b200.synthetic import trajectory


class FakeDataset:
    def __init__(self, n, h=6, w=8):
        self.n, self.h, self.w = n, h, w
        self.poses = [torch.from_numpy(p) for p in trajectory(max(n, 1))][:n]

    def __len__(self):
        return self.n

    def __getitem__(self, i):
        rgb = torch.full((self.h, self.w, 3), i / 100.0)
        depth = torch.full((self.h, self.w), 1.0 + i)
        return i, rgb, depth, self.poses[i]

    def __iter__(self):
        return (self[i] for i in range(self.n))

    def get_camera(self):
        return Camera(4.0, 4.0, 3.5, 2.5, self.w, self.h)


class RecordingAlgorithm:
    """The Algorithm interface the run uses; every call is logged."""

    def __init__(self, separate_LR=False, rot_rep='axis_angle'):
        self.log, self.est, self.gt, self.gt_ori = [], [], [], []
        self.initialized, self.sep, self.rot = False, separate_LR, rot_rep

    device = 'cpu'

    def get_estimate_c2w_list(self):
        return self.est

    def is_separate_LR(self):
        return self.sep

    def get_rot_rep(self):
        return self.rot

    def is_initialized(self):
        return self.initialized

    def seed_frame_tensors(self, frame, rgb=None, depth=None):
        assert float(depth[0, 0]) == 1.0 + frame.fid
        self.log.append(('seed', frame.fid))

    def do_tracking(self, frame):
        self.log.append(('track', frame.fid))
        if self.initialized:
            pose = frame.get_pose().detach().numpy().copy()
            pose[:3, 3] += 0.01
            return pose

    def add_framepose(self, c2w, gt_c2w, gt_c2w_ori):
        self.log.append(('add_framepose', len(self.est)))
        self.est.append(c2w)
        self.gt.append(gt_c2w)
        self.gt_ori.append(gt_c2w_ori)

    def do_mapping(self, frame):
        self.log.append(('map', frame.fid, frame.is_final_frame))
        self.initialized = True

    def update_framepose(self, fid, c2w):
        self.log.append(('update_framepose', fid))
        self.est[fid] = c2w

    def add_keyframe(self, frame):
        self.log.append(('keyframe', frame.fid))

    def finish_frame(self, frame):
        self.log.append(('finish', frame.fid))

    def eval_re_render(self, dataset, render_freq=50):
        self.log.append(('eval_re_render', render_freq))
        return {'frames': []}

    def save_final_mesh(self, out_dir, dataset):
        self.log.append(('save_final_mesh',))

    def save_eval(self, out_dir, idx):
        self.log.append(('save_eval', idx))

    def set_finished(self):
        self.log.append(('set_finished',))


def expected_calls(n, map_every, keyframe_every, lazy_start=-1):
    """tracker.spin + mapper.spin restated: the order the blocking map_buffer / events give."""
    calls, initialized = [], False
    for fid in range(n):
        calls += [('seed', fid), ('track', fid), ('add_framepose', fid)]
        every = 1 if fid <= lazy_start else map_every
        if every != -1 and (fid % every == 0 or fid == n - 1):
            calls += [('map', fid, fid == n - 1), ('update_framepose', fid)]
            if fid % keyframe_every == 0:
                calls.append(('keyframe', fid))
        calls.append(('finish', fid))
    return calls


def _run(tmp_path, n, tracker, keyframe_every, render_freq=50):
    cfg = P.XRDSLAMConfig(out_dir=tmp_path, tracker=P.TrackerConfig(**tracker),
                          mapper=P.MapperConfig(keyframe_every=keyframe_every))
    cfg.tracker.render_freq = render_freq
    algo = RecordingAlgorithm()
    res = P.XRDSLAM(cfg, dataset=FakeDataset(n), algorithm=algo).run()
    return algo, res


SCHEDULES = [(name, p['tracker'], p['mapper']['keyframe_every']) for name, p in P.PRESETS.items()]
SCHEDULES += [('map_every=-1', dict(map_every=-1), 5),
              ('lazy_start=4', dict(map_every=5, lazy_start=4), 3)]


@pytest.mark.parametrize('n', [0, 1, 2, 23])
@pytest.mark.parametrize('schedule', range(len(SCHEDULES)))
def test_call_sequence(tmp_path, n, schedule):
    _, tracker, ke = SCHEDULES[schedule]
    algo, res = _run(tmp_path, n, tracker, ke)
    exp = expected_calls(n, tracker.get('map_every', 1), ke, tracker.get('lazy_start', -1))
    if n > 0:
        exp += [('eval_re_render', 50), ('save_final_mesh',), ('save_eval', n - 1)]
    exp.append(('set_finished',))
    assert algo.log == exp
    assert res['n_frames'] == n and len(algo.est) == n


def test_final_frame_flag_only_on_last_map_frame(tmp_path):
    algo, _ = _run(tmp_path, 23, dict(map_every=5), 5)
    maps = [c for c in algo.log if c[0] == 'map']
    assert [c[1] for c in maps] == [0, 5, 10, 15, 20, 22]
    assert [c[2] for c in maps] == [False] * 5 + [True]


def test_tracked_pose_is_used_once_initialised(tmp_path):
    algo, _ = _run(tmp_path, 3, dict(map_every=1), 1)
    ds = FakeDataset(3)
    # frame 0: not initialised before its mapping -> its ground-truth pose
    assert np.allclose(algo.est[0].numpy(), ds.poses[0].numpy(), atol=1e-5)
    # frame 1: predicted from frame 0, then the tracker's candidate (+0.01 in translation)
    exp = algo.est[0].numpy().copy()
    exp[:3, 3] += 0.01
    assert np.allclose(algo.est[1].numpy(), exp, atol=1e-5)


def _predict_f64(fid, gt, est):
    if fid < 1:
        return gt
    if fid == 1:
        return est[0]
    prev2, prev = est[fid - 2], est[fid - 1]
    return (prev @ np.linalg.inv(prev2)) @ prev


def test_predict_current_pose_matches_f64():
    poses = trajectory(5)
    est = [torch.from_numpy(p) for p in poses]
    for fid in range(5):
        got = P.predict_current_pose(fid, poses[fid], est)
        ref = _predict_f64(fid, poses[fid].astype(np.float64),
                           [p.astype(np.float64) for p in poses])
        assert got.dtype == np.float32 if fid >= 1 else got is poses[fid]
        assert np.allclose(got, ref, atol=2e-6)


def test_relative_pose_matches_f64():
    poses = trajectory(4)
    state = {}
    out = [P.relative_pose(i, poses[i], state, 10) for i in range(4)]
    new0 = np.eye(4)
    new0[:3, 3] += 10
    assert np.array_equal(out[0], new0)
    inv0 = np.linalg.inv(poses[0].astype(np.float64))
    for i in range(1, 4):
        ref = new0 @ (inv0 @ poses[i].astype(np.float64))
        assert out[i].dtype == np.float64 and np.allclose(out[i], ref, atol=1e-6)


@pytest.mark.parametrize('flag', ['enable_vis', 'save_debug_result', 'save_gt_mesh'])
def test_out_of_scope_flags_raise(flag):
    cfg = P.XRDSLAMConfig()
    if flag == 'enable_vis':
        cfg.enable_vis = True
    else:
        setattr(cfg.tracker, flag, True)
    with pytest.raises(NotImplementedError):
        P.XRDSLAM(cfg, dataset=FakeDataset(1), algorithm=RecordingAlgorithm())


def test_presets_apply_and_match_package_defaults():
    for method, p in P.PRESETS.items():
        cfg = P.make_config(method)
        assert cfg.algorithm_name == method
        assert cfg.tracker == P.TrackerConfig(**p['tracker'])
        assert cfg.mapper.keyframe_every == p['mapper']['keyframe_every']
        for k, v in p['algorithm_values'].items():
            assert getattr(cfg.algorithm, k) == v, (method, k)
        for k, v in p['model_values'].items():
            assert getattr(cfg.algorithm.model, k) == v, (method, k)
        for k, v in p['mesher_values'].items():
            assert getattr(cfg.algorithm.mesher, k) == v, (method, k)
        for k in p['pretrained']:
            assert getattr(cfg.algorithm.model, k) is None, (method, k)


# Every preset value that differs from the package's defaults, and the values not carried.
EXPECTED_DIFFERENCES = {
    'nice-slam': {'model': {'points_batch_size': (100000, 500000)},
                  'not_carried': {'pretrained_decoders_coarse': 'pretrained/nice_slam/coarse.pt',
                                  'pretrained_decoders_middle_fine':
                                  'pretrained/nice_slam/middle_fine.pt'}},
    'vox-fusion': {},
    'co-slam': {},
    'point-slam': {'model': {'points_batch_size': (500000, 50000)},
                   'not_carried': {'pretrained_decoders_middle_fine':
                                   'pretrained/point_slam/middle_fine.pt', 'cuda_id': 0}},
}


def test_preset_differences_are_listed():
    for method in P.PRESETS:
        got = {k: v for k, v in P.preset_differences(method).items() if v}
        assert got == EXPECTED_DIFFERENCES[method], method


def test_pretrained_decoder_paths_reach_the_model_config():
    cfg = P.make_config('nice-slam', pretrained_decoders_coarse='a/coarse.pt',
                        pretrained_decoders_middle_fine='a/middle_fine.pt')
    assert str(cfg.algorithm.model.pretrained_decoders_coarse) == 'a/coarse.pt'
    assert str(cfg.algorithm.model.pretrained_decoders_middle_fine) == 'a/middle_fine.pt'
    cfg = P.make_config('point-slam', pretrained_decoders_middle_fine='b.pt')
    assert str(cfg.algorithm.model.pretrained_decoders_middle_fine) == 'b.pt'
    with pytest.raises(ValueError):
        P.make_config('co-slam', pretrained_decoders_coarse='a/coarse.pt')


def _reference_presets(path):
    """tracker / mapper keywords and the algorithm config's literal keywords of every
    XRDSLAMerConfig in the reference's input_config.py, read with ast (nothing is imported)."""
    tree = ast.parse(open(path).read())
    out = {}
    for node in ast.walk(tree):
        if not (isinstance(node, ast.Assign) and isinstance(node.value, ast.Call)):
            continue
        tgt = node.targets[0]
        if not (isinstance(tgt, ast.Subscript) and isinstance(tgt.slice, ast.Constant)):
            continue
        name, calls = tgt.slice.value, {}
        for sub in ast.walk(node.value):
            if isinstance(sub, ast.Call) and isinstance(sub.func, ast.Name):
                kws = {}
                for kw in sub.keywords:
                    v = kw.value
                    if (isinstance(v, ast.Call) and isinstance(v.func, ast.Name)
                            and v.func.id == 'Path'):
                        kws[kw.arg] = ('Path', v.args[0].value)
                        continue
                    try:
                        kws[kw.arg] = ast.literal_eval(v)
                    except ValueError:
                        pass
                calls.setdefault(sub.func.id, kws)
        out[name] = calls
    return out


@pytest.mark.needs_reference
def test_presets_equal_reference_input_config():
    from oracle import ref_harness
    path = os.path.join(ref_harness.REF_ROOT, 'slam', 'configs', 'input_config.py')
    ref = _reference_presets(path)
    for method, p in P.PRESETS.items():
        calls = ref[method]
        assert calls['TrackerConfig'] == p['tracker'], method
        assert calls['MapperConfig'] == p['mapper'], method
        algo = calls[p['algorithm'].split('.')[1]]
        for k, v in p['algorithm_values'].items():
            assert algo[k] == v, (method, k)
        # the model and mesher configs' literal keywords: carried, or listed as not carried
        model = calls[MODEL_CALL[method]]
        assert {k: v for k, v in model.items() if not isinstance(v, tuple)} == \
            {**p['model_values'], **p.get('not_carried', {})}, method
        assert {k: v[1] for k, v in model.items() if isinstance(v, tuple)} == p['pretrained']
        assert calls.get('MesherConfig', {}) == p['mesher_values'], method


MODEL_CALL = {'nice-slam': 'ConvOnetConfig', 'vox-fusion': 'SparseVoxelConfig',
              'co-slam': 'JointEncodingConfig', 'point-slam': 'ConvOnet2Config'}


def test_replica_reader_host_part(tmp_path):
    from xrdslam_b200.datasets import Replica
    res = tmp_path / 'results'
    res.mkdir()
    for k in (2, 0, 1):  # created out of order: the reader sorts
        (res / f'frame{k:06d}.jpg').write_bytes(b'')
        (res / f'depth{k:06d}.png').write_bytes(b'')
    rng = np.random.default_rng(0)
    raw = rng.normal(size=(3, 4, 4))
    raw[:, 3] = [0, 0, 0, 1]
    with open(tmp_path / 'traj.txt', 'w') as f:
        for m in raw:
            f.write(' '.join(repr(float(v)) for v in m.reshape(-1)) + '\n')
    with open(tmp_path / 'devices.yaml', 'w') as f:
        f.write('cam:\n  H: 680\n  W: 1200\n  fx: 600.0\n  fy: 601.0\n  cx: 599.5\n'
                '  cy: 339.5\n  png_depth_scale: 6553.5\n  crop_edge: 7\n'
                '  downsample_factor: 3\n  distortion: [0.1, -0.2, 0.001, 0.002, 0.05]\n')
    ds = Replica(str(tmp_path), device='cpu')
    assert len(ds) == 3
    assert [os.path.basename(p) for p in ds.color_paths] == [f'frame{k:06d}.jpg' for k in range(3)]
    assert [os.path.basename(p) for p in ds.depth_paths] == [f'depth{k:06d}.png' for k in range(3)]
    c = ds.camera
    assert (c.fx, c.fy) == (600.0 / 3, 601.0 / 3)
    assert (c.cx, c.cy) == ((599.5 - 7) / 3, (339.5 - 7) / 3)
    assert (c.height, c.width) == (int((680 - 14) / 3), int((1200 - 14) / 3)) == (222, 395)
    assert ds.crop_edge == 7 and ds.downsample_factor == 3 and ds.png_depth_scale == 6553.5
    assert np.array_equal(ds.distortion, [0.1, -0.2, 0.001, 0.002, 0.05])
    for k in range(3):
        exp = raw[k].copy()
        exp[:3, 1] *= -1
        exp[:3, 2] *= -1
        assert ds.poses[k].dtype == torch.float32
        assert torch.equal(ds.poses[k], torch.from_numpy(exp).float())
