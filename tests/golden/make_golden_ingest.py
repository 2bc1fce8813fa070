"""Write tests/golden/ingest_ref.npz: the reference's frame transform (slam/common/datasets.py:
95-134, BaseDataset.__getitem__ after the two imreads) run with the real cv2 calls it makes, on
small seeded raw frames, so that oracle/ingest.py (and through it csrc/ingest.cu) is pinned to
cv2 itself.

    python tests/golden/make_golden_ingest.py

Each case is run three times: with cv2's defaults (`<case>/rgb`, `<case>/depth`: with Intel
IPP, as a reference run of a cv2 wheel built with IPP executes it), with IPP switched off
(`<case>/rgb_noipp`, `<case>/depth_noipp`: cv2.ipp.setUseIPP(False), optimisations on) and with
cv2.setUseOptimized(False).  The last two run cv2's own C++ code; the script checks that they
agree bit for bit and stores them once.  Stored per case: the inputs (uint8 BGR colour as cv2.imread returns it,
uint16 depth), the camera row (fx, fy, cx, cy, png_depth_scale, crop_edge, downsample_factor) and
the distortion coefficients (empty = none).  `meta` holds the cv2 and IPP versions."""
import json
import os

import cv2
import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, 'ingest_ref.npz')

# Replica's devices.yaml (1200 x 680, fx = fy = 600, cx = 599.5, cy = 339.5, png_depth_scale
# 6553.5) at a tenth of its size; ScanNet-like colour 1296 x 968 over depth 640 x 480, also at a
# tenth.  (name, colour H0 x W0, depth Hd x Wd, fx, fy, cx, cy, scale, crop_edge, downsample, dist)
TUM_DIST = [0.2624, -0.9531, -0.0054, 0.0026, 1.1633]
CASES = [
    ('identity', (68, 120), (68, 120), 60.0, 60.0, 59.95, 33.95, 6553.5, 0, 1, None),
    ('colour_larger', (97, 130), (48, 64), 116.9, 117.4, 64.8, 48.6, 1000.0, 0, 1, None),
    ('crop', (68, 120), (68, 120), 60.0, 60.0, 59.95, 33.95, 6553.5, 5, 1, None),
    ('down2_odd', (51, 75), (51, 75), 40.0, 41.0, 37.0, 25.0, 5000.0, 0, 2, None),
    ('down3_odd', (53, 77), (53, 77), 40.0, 41.0, 38.0, 26.0, 5000.0, 0, 3, None),
    ('down2_even', (60, 80), (60, 80), 52.5, 52.5, 39.5, 29.5, 6553.5, 0, 2, None),
    ('distortion5', (60, 80), (60, 80), 51.7, 51.6, 31.8, 25.4, 5000.0, 0, 1, TUM_DIST),
    ('combined', (97, 131), (49, 65), 116.9, 117.4, 64.8, 48.6, 1000.0, 3, 3, TUM_DIST),
]


def reference_transform(color_data, depth_data, fx, fy, cx, cy, png_depth_scale, crop_edge,
                        downsample_factor, distortion):
    """datasets.py:103-134 verbatim in its calls: cv2 and numpy as the dataset makes them."""
    if distortion is not None:
        K = np.array([[fx, 0.0, cx], [0.0, fy, cy], [0.0, 0.0, 1.0]])
        color_data = cv2.undistort(color_data, K, np.array(distortion))
    color_data = cv2.cvtColor(color_data, cv2.COLOR_BGR2RGB)
    color_data = color_data / 255.
    depth_data = depth_data.astype(np.float32) / png_depth_scale
    H, W = depth_data.shape
    color_data = cv2.resize(color_data, (W, H))
    edge = crop_edge
    if edge > 0:
        color_data = color_data[edge:-edge, edge:-edge]
        depth_data = depth_data[edge:-edge, edge:-edge]
    if downsample_factor > 1:
        H = (H - 2 * edge) // downsample_factor
        W = (W - 2 * edge) // downsample_factor
        color_data = cv2.resize(color_data, (W, H), interpolation=cv2.INTER_LINEAR)
        depth_data = cv2.resize(depth_data, (W, H), interpolation=cv2.INTER_NEAREST)
    return (torch.from_numpy(color_data).to(torch.float).numpy(),
            torch.from_numpy(depth_data).to(torch.float).numpy())


def raw_frames(shape_c, shape_d, seed):
    """Seeded colour (smooth ramps plus noise, so every interpolation weight matters) and depth
    (uint16 over the full range, 3 % zeros)."""
    rng = np.random.default_rng(seed)
    H0, W0 = shape_c
    yy, xx = np.mgrid[0:H0, 0:W0]
    ramp = np.stack([xx * 255.0 / W0, yy * 255.0 / H0, (xx + yy) * 127.0 / (W0 + H0)], -1)
    color = np.clip(ramp + rng.normal(0, 40, (H0, W0, 3)), 0, 255).astype(np.uint8)
    depth = rng.integers(0, 65536, shape_d, dtype=np.uint16)
    depth[rng.random(shape_d) < 0.03] = 0
    return color, depth


def main():
    out = {}
    for k, (name, sc, sd, fx, fy, cx, cy, scale, edge, f, dist) in enumerate(CASES):
        color, depth = raw_frames(sc, sd, seed=100 + k)
        args = (fx, fy, cx, cy, scale, edge, f, dist)
        cv2.setUseOptimized(True)      # also switches IPP back on
        rgb, dep = reference_transform(color.copy(), depth.copy(), *args)
        cv2.ipp.setUseIPP(False)
        rgb_n, dep_n = reference_transform(color.copy(), depth.copy(), *args)
        cv2.setUseOptimized(False)
        rgb_g, dep_g = reference_transform(color.copy(), depth.copy(), *args)
        cv2.setUseOptimized(True)
        out[f'{name}/color'] = color
        out[f'{name}/depth_u16'] = depth
        out[f'{name}/camera'] = np.array([fx, fy, cx, cy, scale, edge, f], np.float64)
        out[f'{name}/dist'] = np.array(dist if dist is not None else [], np.float64)
        out[f'{name}/rgb'], out[f'{name}/depth'] = rgb, dep
        assert np.array_equal(rgb_n.view(np.int32), rgb_g.view(np.int32)), name
        assert np.array_equal(dep_n.view(np.int32), dep_g.view(np.int32)), name
        out[f'{name}/rgb_noipp'], out[f'{name}/depth_noipp'] = rgb_n, dep_n
    out['meta'] = np.array(json.dumps({'cv2': cv2.__version__, 'ipp': cv2.ipp.getIppVersion(),
                                       'cases': [c[0] for c in CASES]}))
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), 'bytes')


if __name__ == '__main__':
    main()
