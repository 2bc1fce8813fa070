"""Time the ds-eval reconstruction metrics on the device (csrc/eval.cu) beside scipy's cKDTree.

Reports, with the card name and power limit: nearest-neighbour index build time and query rate
for 200k/200k and 2M/2M points on the synthetic room's surface with 0 %, 1 % and 10 % outliers
0.5-3 m off it, with the octree nodes entered and points tested per query; one ICP iteration;
calc_3d_metric and the F-score path end to end; cKDTree(workers=-1) on the same points.
Prints one JSON line per measurement and, with --out, writes them all to <out>/time_eval.json.

    python scripts/time_eval.py [--out DIR] [--sizes 200000 2000000]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import eval_recon as oe  # noqa: E402
from xrdslam_b200 import _cabi, io_formats  # noqa: E402
from xrdslam_b200 import eval_recon as er  # noqa: E402
from xrdslam_b200.synthetic import room_mesh  # noqa: E402


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f'unknown ({e})'


def cuda_ms(fn, reps=3):
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


def points(n, outlier_frac, seed, dev):
    v, f = room_mesh(0.1)
    p, _ = er.sample_surface(v, f, n, 0, None, seed, dev)
    k = int(n * outlier_frac)
    if k:
        g = torch.Generator(device=dev).manual_seed(seed)
        d = torch.randn(k, 3, device=dev, generator=g)
        d = d / d.norm(dim=1, keepdim=True)
        p[:k] += d * (0.5 + 2.5 * torch.rand(k, 1, device=dev, generator=g))
    return p


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--sizes', type=int, nargs='+', default=[200000, 2000000])
    a = ap.parse_args()
    dev = torch.device('cuda:0')
    rows = [dict(card=card())]
    for n in a.sizes:
        tgt = points(n, 0.0, 1, dev)
        for frac in (0.0, 0.01, 0.1):
            q = points(n, frac, 2, dev)
            build = cuda_ms(lambda: er.NNIndex(tgt, dev))
            idx = er.NNIndex(tgt, dev)
            qms = cuda_ms(lambda: idx.query(q))
            cnt = torch.zeros(2, dtype=torch.int64, device=dev)
            _cabi.lib().xrd_debug_nn_counters(cnt.data_ptr())
            idx.query(q)
            torch.cuda.synchronize()
            _cabi.lib().xrd_debug_nn_counters(None)
            nodes, pts = cnt.tolist()
            from scipy.spatial import cKDTree
            P, Q = tgt.double().cpu().numpy(), q.double().cpu().numpy()
            t0 = time.perf_counter()
            tree = cKDTree(P)
            t1 = time.perf_counter()
            tree.query(Q, workers=-1)
            t2 = time.perf_counter()
            rows.append(dict(what='nn', n_target=n, n_query=n, outliers=frac,
                             build_ms=round(build, 3), query_ms=round(qms, 3),
                             queries_per_s=round(n / qms * 1e3),
                             nodes_per_query=round(nodes / n, 2),
                             points_per_query=round(pts / n, 2),
                             ckdtree_build_ms=round((t1 - t0) * 1e3, 1),
                             ckdtree_query_ms=round((t2 - t1) * 1e3, 1)))
            print(json.dumps(rows[-1]), flush=True)
    # ICP iteration on the room's vertices at 1 cm spacing
    gv, gf = room_mesh(0.01)
    g = torch.from_numpy(gv).to(dev)
    T = np.eye(4)
    T[:3, 3] = [0.02, -0.01, 0.01]
    src = er.transform(g, T)
    idx = er.NNIndex(g, dev)
    one = cuda_ms(lambda: er.registration_icp(src, idx, 0.1, max_iteration=1))
    rows.append(dict(what='icp', n=len(gv), one_iteration_ms_incl_setup=round(one, 3)))
    print(json.dumps(rows[-1]), flush=True)
    # end to end on the room mesh against itself, shifted
    with tempfile.TemporaryDirectory() as d:
        rv = oe.transform(gv, T)
        rec = io_formats.write_ply(os.path.join(d, 'final_mesh_rec.ply'), rv, gf)
        gtp = io_formats.write_ply(os.path.join(d, 'gt.ply'), gv, gf)
        t3 = cuda_ms(lambda: er.calc_3d_metric(rec, gtp, transform_matrix=np.eye(4)), reps=2)
        tf = cuda_ms(lambda: er.calc_3d_metric_New(rec, gtp, transform_matrix=np.eye(4)), reps=2)
    rows.append(dict(what='end_to_end', n_vertices=len(gv), calc_3d_metric_ms=round(t3, 1),
                     fscore_path_ms=round(tf, 1)))
    print(json.dumps(rows[-1]), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, 'time_eval.json'), 'w') as fh:
            json.dump(rows, fh, indent=1)


if __name__ == '__main__':
    main()
