"""xrd_frame_ingest_f32 (float32 OpenEXR depth) bit for bit against the numpy restatement, its
status codes against xrd_frame_ingest's, every dataset layout's device frames against the
restatement on the decoded files, and SLAM runs over synthetic TUM RGB-D and ScanNet folders."""
import math
import os

import numpy as np
import pytest
import torch

from ingest_f32_oracle import ingest_f32
from oracle import ingest as O

pytestmark = pytest.mark.gpu


def _bits_equal(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return a.shape == b.shape and np.array_equal(a.view(np.int32), b.view(np.int32))


def _seeded_f32(B, H, W, seed):
    """Depth in metres with NaN (several payloads, signalling ones too), +-inf, +-0, negative,
    subnormal and large values scattered over it."""
    rng = np.random.default_rng(seed)
    d = rng.uniform(0.0, 8.0, (B, H, W)).astype(np.float32)
    flat = d.reshape(-1)
    specials = np.array([np.nan, np.inf, -np.inf, 0.0, -0.0, -1.25, -7.5, 1e-40, -2e-43, 1e-45,
                         1.1754942e-38, 3.4e38, -3.4e38, 1e30, 65535.0], np.float32)
    idx = rng.choice(flat.size, size=flat.size // 5, replace=False)
    flat[idx] = specials[rng.integers(0, specials.size, idx.size)]
    nan_bits = np.array([0x7fc00000, 0xffc00000, 0x7fc12345, 0x7fa00001, 0x7f800001,
                         0xff812345, 0x7fffffff], np.uint32)
    nidx = rng.choice(flat.size, size=max(flat.size // 50, 7), replace=False)
    flat.view(np.uint32)[nidx] = nan_bits[np.arange(nidx.size) % nan_bits.size]
    return d


def _seeded_color(B, H, W, seed):
    rng = np.random.default_rng(seed)
    return rng.integers(0, 256, (B, H, W, 3), dtype=np.uint8)


def _run(color, depth, dev, *args):
    from xrdslam_b200.datasets import frame_ingest
    c = torch.from_numpy(np.ascontiguousarray(color)).to(dev)
    d = torch.from_numpy(np.ascontiguousarray(depth)).to(dev)
    rgb, dep = frame_ingest(c, d, *args)
    return rgb.cpu().numpy(), dep.cpu().numpy()


DIST5 = [0.2624, -0.9531, -0.0054, 0.0026, 1.1633]
# (H, W, colour scale, png_depth_scale, distortion)
SHAPES = [(97, 131, 1, 1.0, None), (120, 160, 2, 5000.0, None), (61, 83, 1, 6553.5, DIST5),
          (64, 80, 1.5, 1000.0, None)]


@pytest.mark.parametrize('B', [1, 4])
@pytest.mark.parametrize('edge', [0, 3])
@pytest.mark.parametrize('f', [1, 2, 3])
@pytest.mark.parametrize('shape', range(len(SHAPES)))
def test_f32_ingest_bit_exact(cuda_dev, B, edge, f, shape):
    H, W, cs, scale, dist = SHAPES[shape]
    color = _seeded_color(B, int(round(H * cs)), int(round(W * cs)), 100 + shape)
    depth = _seeded_f32(B, H, W, 200 + 10 * shape + f + edge)
    fx, fy, cx, cy = 0.5 * W, 0.52 * W, 0.5 * W - 0.5, 0.5 * H - 0.5
    args = (fx * cs, fy * cs, cx * cs, cy * cs, dist, scale, edge, f)
    rgb, dep = _run(color, depth, cuda_dev, *args)
    for b in range(B):
        orgb, odep = ingest_f32(color[b], depth[b], *args)
        assert _bits_equal(rgb[b], orgb), b
        assert _bits_equal(dep[b], odep), b
    assert np.isnan(dep).any() and np.isinf(dep).any()


def test_f32_nan_scale_and_payloads(cuda_dev):
    """NaN and infinite scales: a NaN scale comes back as that NaN unless the depth is NaN itself,
    inf / inf as x86's default NaN, as numpy divides."""
    depth = _seeded_f32(1, 16, 24, 7)
    color = _seeded_color(1, 16, 24, 8)
    for scale in (float('nan'), -0.5, 1e-30, float('inf'), 1e-50):  # 1e-50: f32 0, 0 / 0
        _, dep = _run(color, depth, cuda_dev, 12., 12., 11.5, 7.5, None, scale, 0, 1)
        _, odep = ingest_f32(color[0], depth[0], 12., 12., 11.5, 7.5, None, scale, 0, 1)
        assert _bits_equal(dep[0], odep), scale


def test_f32_status_codes_match_u16(cuda_dev):
    from xrdslam_b200 import _cabi
    from xrdslam_b200.datasets import ingest_config
    L = _cabi.lib()
    B, H, W = 2, 48, 64
    p = _cabi.ptr
    color = torch.zeros(B, H, W, 3, dtype=torch.uint8, device=cuda_dev)
    d16 = torch.zeros(B, H, W, dtype=torch.int16, device=cuda_dev)
    d32 = torch.zeros(B, H, W, dtype=torch.float32, device=cuda_dev)
    rgb = torch.empty(B, H, W, 3, device=cuda_dev)
    dep = torch.empty(B, H, W, device=cuda_dev)
    cfg = ingest_config(B, (H, W), (H, W), 30.0, 30.0, 32.0, 24.0, DIST5)
    need = L.xrd_frame_ingest_workspace_bytes(cfg)
    ws = torch.empty(need, dtype=torch.uint8, device=cuda_dev)

    def both(c, nbytes, color_p=p(color), ws_p=p(ws), depth_null=False):
        a = L.xrd_frame_ingest(c, color_p, None if depth_null else p(d16), p(rgb), p(dep), ws_p,
                               nbytes, None)
        b = L.xrd_frame_ingest_f32(c, color_p, None if depth_null else p(d32), p(rgb), p(dep),
                                   ws_p, nbytes, None)
        return a, b

    cases = [(cfg, need, {}), (cfg, need - 1, {}), (cfg, need, dict(ws_p=None)),
             (cfg, need, dict(color_p=None)), (cfg, need, dict(depth_null=True)),
             (None, need, {}),
             (ingest_config(B, (H, W), (H, W), 30., 30., 32., 24.), 0, dict(ws_p=None))]
    for bad in (ingest_config(B, (H, W), (H, W), 30., 30., 32., 24., crop_edge=24),
                ingest_config(B, (H, W), (H, W), 30., 30., 32., 24., crop_edge=23,
                              downsample_factor=3),
                ingest_config(B, (H, W), (H, W), 30., 30., 32., 24., DIST5 + [0.0]),
                ingest_config(B, (H, W), (H, W), 30., 30., 32., 24., downsample_factor=0),
                ingest_config(0, (H, W), (H, W), 30., 30., 32., 24.),
                ingest_config(B, (H, W), (H, W), 30., 30., 32., 24., png_depth_scale=0.0)):
        cases.append((bad, need, {}))
    got = [both(c, n, **k) for c, n, k in cases]
    torch.cuda.synchronize()
    assert [a for a, _ in got] == [b for _, b in got]
    assert [a for a, _ in got] == [0, -3, -6, -6, -6, -6, 0] + [-1] * 6


# ---- every layout's device frames ------------------------------------------------------------
W, H = 96, 72
LAYOUTS = [('tumrgbd', 'write_tum', dict(n_frames=4, distortion=DIST5, crop_edge=3)),
           ('scannet', 'write_scannet', dict(n_frames=3, crop_edge=4, downsample_factor=2)),
           ('7scenes', 'write_7scenes', dict(n_frames=3, downsample_factor=3)),
           ('azure', 'write_azure', dict(n_frames=3, distortion=DIST5)),
           ('cofusion', 'write_cofusion', dict(n_frames=3, crop_edge=2, downsample_factor=2))]


@pytest.mark.parametrize('case', range(len(LAYOUTS)))
def test_reader_frames(cuda_dev, tmp_path, case):
    from xrdslam_b200 import synthetic as S
    from xrdslam_b200.datasets import get_dataset, read_color, read_depth_any
    key, writer, kw = LAYOUTS[case]
    getattr(S, writer)(str(tmp_path), width=W, height=H, **kw)
    ds = get_dataset(str(tmp_path), key, device=str(cuda_dev))
    assert len(ds) == kw['n_frames']
    c = ds.camera
    for i in range(len(ds)):
        idx, rgb, depth, c2w = ds[i]
        assert idx == i and rgb.device.type == 'cuda' and depth.device.type == 'cuda'
        assert rgb.shape == (c.height, c.width, 3) and depth.shape == (c.height, c.width)
        color, raw = read_color(ds.color_paths[i]), read_depth_any(ds.depth_paths[i])
        args = (ds.fx, ds.fy, ds.cx, ds.cy, ds.distortion, ds.png_depth_scale, ds.crop_edge,
                ds.downsample_factor)
        orgb, odep = ingest_f32(color, raw, *args) if raw.dtype == np.float32 else \
            O.ingest(color, raw, *args)
        assert _bits_equal(rgb.cpu().numpy(), orgb) and _bits_equal(depth.cpu().numpy(), odep)
        assert torch.equal(c2w.cpu(), ds.poses[i]) and c2w.dtype == torch.float32
    seen = list(ds)
    assert [s[0] for s in seen] == list(range(len(ds)))
    for i, (idx, rgb, depth, c2w) in enumerate(seen):
        _, r2, d2, p2 = ds[i]
        assert _bits_equal(rgb.cpu(), r2.cpu()) and _bits_equal(depth.cpu(), d2.cpu())
        assert torch.equal(c2w, p2)


# ---- SLAM runs over TUM RGB-D and ScanNet folders ---------------------------------------------
N_FRAMES, RUN_W, RUN_H, TURN = 15, 224, 176, 0.05
# as tests/test_pipeline_gpu.py: the presets' tracking iteration counts, fewer mapping iterations
REDUCED = {
    'co-slam': dict(tracking_n_iters=10, mapping_n_iters=5, mapping_first_n_iters=30,
                    mapping_sample=1024),
    'vox-fusion': dict(tracking_n_iters=30, mapping_n_iters=5, mapping_first_n_iters=10),
}
# the synthetic room with a margin (the presets carry Replica office0's bounds)
BOUND = [[-3.2, 3.2], [-4.2, 2.7], [-2.2, 2.7]]
ATE_RATIO = 0.7


@pytest.fixture(scope='module')
def run_folders(tmp_path_factory):
    from xrdslam_b200 import synthetic as S
    tum = str(tmp_path_factory.mktemp('tum_run'))
    S.write_tum(tum, N_FRAMES, width=RUN_W, height=RUN_H, turn=TURN)
    scannet = str(tmp_path_factory.mktemp('scannet_run'))
    S.write_scannet(scannet, N_FRAMES, width=RUN_W, height=RUN_H, turn=TURN, color_scale=2.0,
                    crop_edge=4)
    return {'tumrgbd': tum, 'scannet': scannet}


def _check_run(out, res, cuda_dev, label):
    from xrdslam_b200.eval import EvalMatrics
    from xrdslam_b200.io_formats import ate_rmse, load_eval_tar
    assert res['n_frames'] == N_FRAMES
    for name in ('eval.tar', 'final_mesh.ply', 'final_mesh_rec.ply'):
        assert os.path.exists(os.path.join(out, name)), name
    est, gt_ori, n = load_eval_tar(os.path.join(out, 'eval.tar'))
    assert n == N_FRAMES - 1 and len(est) == N_FRAMES
    ev = EvalMatrics(output_dir=out, eval_recon=False, device=str(cuda_dev))
    ev.main()
    ate = float(ev.traj_result['rmse'])
    frozen = ate_rmse(gt_ori, [gt_ori[0]] * len(gt_ori), n)['rmse']
    print(f'{label}: ATE RMSE {ate:.5f} m ({ate / frozen:.3f} of no motion), '
          f'timing {res["timing"]}')
    assert math.isfinite(ate) and ate < ATE_RATIO * frozen


@pytest.mark.parametrize('data_type', ['tumrgbd', 'scannet'])
@pytest.mark.parametrize('method', ['co-slam', 'vox-fusion'])
def test_run_and_eval(cuda_dev, run_folders, tmp_path, method, data_type):
    import warnings

    from xrdslam_b200.pipeline import XRDSLAM, make_config
    torch.manual_seed(0)
    np.random.seed(0)
    out = str(tmp_path / 'out')
    extra = dict(mapping_bound=BOUND) if method == 'co-slam' else {}
    if method == 'co-slam' and data_type == 'tumrgbd':
        # through the command line: --data_type and --set, nested fields included
        from xrdslam_b200 import run
        sets = {**REDUCED[method], **extra, 'marching_cubes_bound': BOUND,
                'tracker.render_freq': 5}
        argv = [method, '--data', run_folders[data_type], '--data_type', data_type,
                '--out_dir', out, '--device', str(cuda_dev)]
        for k, v in sets.items():
            argv += ['--set', f'{k}={v!r}']
        with warnings.catch_warnings():
            warnings.simplefilter('ignore', UserWarning)
            res = run.main(argv)
    else:
        cfg = make_config(method, data=run_folders[data_type], data_type=data_type,
                          out_dir=out, device=str(cuda_dev), **REDUCED[method], **extra)
        cfg.tracker.render_freq = 5
        with warnings.catch_warnings():
            warnings.simplefilter('ignore', UserWarning)
            res = XRDSLAM(cfg).run()
    assert [r['idx'] for r in res['render']['frames']] == [0, 5, 10]
    _check_run(out, res, cuda_dev, f'{method} on {data_type}')
