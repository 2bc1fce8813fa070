"""xrd_frame_ingest (csrc/ingest.cu) against oracle/ingest.py, bit for bit: the golden cases
recorded with real cv2, seeded full-size frames, the status codes, and the Replica reader on a
synthetic folder."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from oracle import ingest as O

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), 'golden', 'ingest_ref.npz')


def _bits_equal(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return a.shape == b.shape and np.array_equal(a.view(np.int32), b.view(np.int32))


def _run(color, depth, dev, fx, fy, cx, cy, dist, scale, edge, f):
    from xrdslam_b200.datasets import frame_ingest
    c = torch.from_numpy(np.ascontiguousarray(color)).to(dev)
    d = torch.from_numpy(np.ascontiguousarray(depth).view(np.int16)).to(dev)
    rgb, dep = frame_ingest(c, d, fx, fy, cx, cy, dist, scale, edge, f)
    return rgb.cpu().numpy(), dep.cpu().numpy()


def _oracle(color, depth, *args):
    outs = [O.ingest(color[b], depth[b], *args) for b in range(color.shape[0])]
    return np.stack([o[0] for o in outs]), np.stack([o[1] for o in outs])


def test_golden_cases(cuda_dev):
    g = np.load(GOLDEN)
    for name in json.loads(str(g['meta']))['cases']:
        fx, fy, cx, cy, s, e, f = g[name + '/camera']
        dist = g[name + '/dist']
        args = (fx, fy, cx, cy, dist if dist.size else None, s, int(e), int(f))
        rgb, dep = _run(g[name + '/color'][None], g[name + '/depth_u16'][None], cuda_dev, *args)
        orgb, odep = O.ingest(g[name + '/color'], g[name + '/depth_u16'], *args)
        assert _bits_equal(rgb[0], orgb) and _bits_equal(dep[0], odep), name
        assert _bits_equal(rgb[0], g[name + '/rgb_noipp']), name
        assert _bits_equal(dep[0], g[name + '/depth_noipp']), name


def _seeded(B, H, W, seed):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:H, 0:W]
    ramp = np.stack([xx * 255.0 / W, yy * 255.0 / H, (xx + yy) * 127.0 / (W + H)], -1)
    color = np.clip(ramp[None] + rng.normal(0, 30, (B, H, W, 3)), 0, 255).astype(np.uint8)
    depth = rng.integers(0, 65536, (B, H, W), dtype=np.uint16)
    return color, depth


# (H, W, colour scale, crop_edge, downsample_factor, distortion)
DIST5 = [0.2624, -0.9531, -0.0054, 0.0026, 1.1633]
SEEDED = [(680, 1200, 1, 0, 1, None), (680, 1200, 1, 0, 2, DIST5), (680, 1200, 1, 10, 3, None),
          (481, 641, 1, 0, 2, DIST5), (481, 641, 1, 7, 3, None), (481, 641, 2, 0, 1, None),
          (481, 641, 1, 0, 1, [0.01, -0.02, 0.001, 0.0005, 0.0, 0.003, -0.001, 0.0002])]


@pytest.mark.parametrize('B', [1, 4])
@pytest.mark.parametrize('case', range(len(SEEDED)))
def test_seeded_frames(cuda_dev, B, case):
    H, W, cs, edge, f, dist = SEEDED[case]
    color, _ = _seeded(B, H * cs + (cs > 1), W * cs + (cs > 1), 10 + case)
    _, depth = _seeded(B, H, W, 20 + case)
    fx, fy, cx, cy = 0.5 * W * cs, 0.52 * W * cs, 0.5 * W * cs - 0.5, 0.5 * H * cs - 0.5
    args = (fx, fy, cx, cy, dist, 6553.5, edge, f)
    rgb, dep = _run(color, depth, cuda_dev, *args)
    orgb, odep = _oracle(color, depth, *args)
    assert _bits_equal(rgb, orgb) and _bits_equal(dep, odep)


def test_status_codes(cuda_dev):
    from xrdslam_b200 import _cabi
    from xrdslam_b200.datasets import ingest_config
    L = _cabi.lib()
    B, H, W = 2, 48, 64
    color = torch.zeros(B, H, W, 3, dtype=torch.uint8, device=cuda_dev)
    depth = torch.zeros(B, H, W, dtype=torch.int16, device=cuda_dev)
    rgb = torch.empty(B, H, W, 3, device=cuda_dev)
    dep = torch.empty(B, H, W, device=cuda_dev)
    p = _cabi.ptr
    cfg = ingest_config(B, (H, W), (H, W), 30.0, 30.0, 32.0, 24.0, DIST5)
    need = L.xrd_frame_ingest_workspace_bytes(cfg)
    assert need >= B * H * W * 3
    ws = torch.empty(need, dtype=torch.uint8, device=cuda_dev)
    call = lambda c, nbytes, **k: L.xrd_frame_ingest(
        c, k.get('color', p(color)), p(depth), p(rgb), p(dep), k.get('ws', p(ws)), nbytes, None)
    assert call(cfg, need) == 0
    assert call(cfg, need - 1) == -3                      # XRD_E_WORKSPACE
    assert call(cfg, need, ws=None) == -6                 # XRD_E_NULL
    assert call(cfg, need, color=None) == -6
    assert L.xrd_frame_ingest(None, p(color), p(depth), p(rgb), p(dep), p(ws), need, None) == -6
    nodist = ingest_config(B, (H, W), (H, W), 30.0, 30.0, 32.0, 24.0)
    assert L.xrd_frame_ingest_workspace_bytes(nodist) == 0
    assert call(nodist, 0, ws=None) == 0
    for bad in (ingest_config(B, (H, W), (H, W), 30., 30., 32., 24., crop_edge=24),
                ingest_config(B, (H, W), (H, W), 30., 30., 32., 24., crop_edge=23,
                              downsample_factor=3),
                ingest_config(B, (H, W), (H, W), 30., 30., 32., 24., DIST5 + [0.0]),
                ingest_config(B, (H, W), (H, W), 30., 30., 32., 24., downsample_factor=0),
                ingest_config(0, (H, W), (H, W), 30., 30., 32., 24.),
                ingest_config(B, (H, W), (H, W), 30., 30., 32., 24., png_depth_scale=0.0)):
        assert call(bad, need) == -1                      # XRD_E_SHAPE
        assert L.xrd_frame_ingest_workspace_bytes(bad) == 0
    torch.cuda.synchronize()
    from xrdslam_b200.datasets import frame_ingest
    with pytest.raises(ValueError):
        frame_ingest(color, depth, 30., 30., 32., 24., crop_edge=24)


@pytest.fixture(scope='module')
def replica_folder(tmp_path_factory):
    from xrdslam_b200.synthetic import write_replica
    folder = tmp_path_factory.mktemp('replica')
    write_replica(str(folder), 5, width=224, height=176)
    return str(folder)


def test_replica_reader(cuda_dev, replica_folder):
    from xrdslam_b200.datasets import Replica, read_color, read_depth
    ds = Replica(replica_folder, device=str(cuda_dev))
    assert len(ds) == 5
    c = ds.camera
    for i in range(len(ds)):
        idx, rgb, depth, c2w = ds[i]
        assert idx == i and rgb.device.type == 'cuda' and depth.device.type == 'cuda'
        assert rgb.shape == (c.height, c.width, 3) and depth.shape == (c.height, c.width)
        orgb, odep = O.ingest(read_color(ds.color_paths[i]), read_depth(ds.depth_paths[i]),
                              ds.fx, ds.fy, ds.cx, ds.cy, ds.distortion, ds.png_depth_scale,
                              ds.crop_edge, ds.downsample_factor)
        assert _bits_equal(rgb.cpu().numpy(), orgb) and _bits_equal(depth.cpu().numpy(), odep)
        assert torch.equal(c2w.cpu(), ds.poses[i]) and c2w.dtype == torch.float32
    seen = list(ds)
    assert [s[0] for s in seen] == list(range(5))
    for i, (idx, rgb, depth, c2w) in enumerate(seen):
        _, r2, d2, p2 = ds[i]
        assert torch.equal(rgb, r2) and torch.equal(depth, d2) and torch.equal(c2w, p2)
