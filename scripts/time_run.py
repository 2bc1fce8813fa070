"""Time the frame ingest (csrc/ingest.cu) and whole runs (pipeline.XRDSLAM).

Reports, with the card name, power limit and SM clock read in the same call:
  * xrd_frame_ingest for B = 1 and B = 8 seeded frames of 1200 x 680, identity (Replica) and with
    five distortion coefficients plus downsample 2 (best of N, CUDA events, device-resident
    inputs);
  * the host path it replaces for the same frames: the reference's cv2 / numpy calls when cv2 is
    importable, and the numpy oracle (oracle/ingest.py);
  * XRDSLAM(config).run() per algorithm on the synthetic 15-frame Replica folder of 224 x 176 and
    the iteration counts of tests/test_pipeline_gpu.py, in frames/s, split into ingest,
    tracking, mapping and the final pass (device synchronised at phase boundaries).
Prints one JSON line per measurement and, with --out, writes them to <out>/time_run.json.

    python scripts/time_run.py [--out DIR] [--reps N]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from oracle import ingest as oi  # noqa: E402
from xrdslam_b200.datasets import frame_ingest  # noqa: E402

DIST5 = [0.2624, -0.9531, -0.0054, 0.0026, 1.1633]
H, W = 680, 1200
CAM = (600.0, 600.0, 599.5, 339.5)
CASES = {'identity': dict(distortion=None, downsample_factor=1),
         'distortion_down2': dict(distortion=DIST5, downsample_factor=2)}


def card():
    q = 'name,power.limit,clocks.sm,clocks.max.sm'
    try:
        return subprocess.run(['nvidia-smi', f'--query-gpu={q}', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f'unknown ({e})'


def cuda_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    best = float('inf')
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        best = min(best, a.elapsed_time(b))
    return best


def host_ms(fn, reps):
    best = float('inf')
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        best = min(best, (time.perf_counter() - t0) * 1e3)
    return best


def ingest_rows(dev, reps):
    rng = np.random.default_rng(0)
    rows = []
    for B in (1, 8):
        color = rng.integers(0, 256, (B, H, W, 3), dtype=np.uint8)
        depth = rng.integers(0, 65536, (B, H, W), dtype=np.uint16)
        c = torch.from_numpy(color).to(dev)
        d = torch.from_numpy(depth.view(np.int16)).to(dev)
        for name, kw in CASES.items():
            args = dict(png_depth_scale=6553.5, crop_edge=0, **kw)
            ms = cuda_ms(lambda: frame_ingest(c, d, *CAM, **args), reps)
            oracle = host_ms(lambda: [oi.ingest(color[b], depth[b], *CAM, kw['distortion'],
                                                6553.5, 0, kw['downsample_factor'])
                                      for b in range(B)], max(1, reps // 10))
            row = {'what': 'xrd_frame_ingest', 'case': name, 'B': B, 'H': H, 'W': W,
                   'device_ms': ms, 'numpy_oracle_host_ms': oracle}
            try:
                import cv2  # noqa: F401
                from golden.make_golden_ingest import reference_transform
                row['cv2_host_ms'] = host_ms(
                    lambda: [reference_transform(color[b], depth[b], *CAM, 6553.5, 0,
                                                 kw['downsample_factor'], kw['distortion'])
                             for b in range(B)], max(1, reps // 10))
            except ImportError:
                row['cv2_host_ms'] = None
            rows.append(row)
    return rows


def run_rows(dev):
    from test_pipeline_gpu import HEIGHT, N_FRAMES, REDUCED, TURN, WIDTH
    from xrdslam_b200.pipeline import XRDSLAM, make_config
    from xrdslam_b200.synthetic import write_replica
    rows = []
    with tempfile.TemporaryDirectory() as tmp:
        data = os.path.join(tmp, 'replica')
        write_replica(data, N_FRAMES, width=WIDTH, height=HEIGHT, turn=TURN)
        for method, red in REDUCED.items():
            torch.manual_seed(0)
            np.random.seed(0)
            cfg = make_config(method, data=data, out_dir=os.path.join(tmp, method),
                              device=str(dev), **red)
            cfg.profile = True
            cfg.tracker.render_freq = 5
            with warnings.catch_warnings():
                warnings.simplefilter('ignore')
                t0 = time.perf_counter()
                res = XRDSLAM(cfg).run()
                wall = time.perf_counter() - t0
            t = res['timing']
            loop = t['ingest'] + t['tracking'] + t['mapping']
            rows.append({'what': 'XRDSLAM.run', 'method': method, 'frames': N_FRAMES,
                         'size': f'{WIDTH}x{HEIGHT}', 'iterations': red,
                         'frames_per_s': N_FRAMES / loop, 'timing_s': t, 'wall_s': wall})
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out')
    ap.add_argument('--reps', type=int, default=20)
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    rows = [{'what': 'card', 'nvidia-smi': card()}]
    rows += ingest_rows(dev, args.reps)
    rows += run_rows(dev)
    rows.append({'what': 'card', 'nvidia-smi': card()})
    for r in rows:
        print(json.dumps(r))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'time_run.json'), 'w') as f:
            json.dump(rows, f, indent=1)


if __name__ == '__main__':
    main()
