"""Time ds-eval's depth-L1 metric on the device (csrc/eval_render.cu).

Reports, with the card name and power limit: depth-render time per view and triangle-views/s
for the synthetic room at 1 cm (3.86 M faces) and 5 cm (154 k faces) spacing with 1, 8 and 32
views per launch, and the share of (face, view) pairs that take the queued path; the unseen
check for 4096 candidates against 1 M points; calc_2d_metric end to end with 1000 views; the
numpy oracle's time for one 500 x 500 view, for scale.  Prints one JSON line per measurement
and, with --out, writes them all to <out>/time_eval_2d.json.

    python scripts/time_eval_2d.py [--out DIR]
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

from oracle import eval_render as ore  # noqa: E402
from time_eval import card, cuda_ms  # noqa: E402
from xrdslam_b200 import _cabi, io_formats  # noqa: E402
from xrdslam_b200 import eval_recon as er  # noqa: E402
from xrdslam_b200.synthetic import room_mesh  # noqa: E402


def views(v, n, seed):
    ext, T = er.get_cam_position(v)
    return er.sample_views(None, ext, T, n, seed=seed, seen_fn=lambda c: np.zeros(len(c), bool))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    dev = torch.device('cuda:0')
    rows = [dict(card=card())]
    c2w = None
    for spacing in (0.01, 0.05):
        v, f = room_mesh(spacing)
        c2w = views(v, 32, 1)
        w2c = torch.from_numpy(np.linalg.inv(c2w)[:, :3].copy()).to(dev)
        r = er.DepthRenderer(v, f, dev)
        for B in (1, 8, 32):
            out = torch.empty(B, 500, 500, device=dev)
            ms = cuda_ms(lambda: r.render(w2c[:B], out=out), reps=5)
            q = torch.zeros(1, dtype=torch.int32, device=dev)
            _cabi.lib().xrd_debug_eval_render_queued(r.ws.data_ptr(), q.data_ptr(), None)
            rows.append(dict(what='render', faces=len(f), views_per_launch=B,
                             ms_per_view=round(ms / B, 3),
                             triangle_views_per_s=round(len(f) * B / ms * 1e3),
                             queued_share=round(int(q.item()) / (len(f) * B), 5)))
            print(json.dumps(rows[-1]), flush=True)
    # unseen check: 4096 candidates against 1 M points on the walls
    pts, _ = er.sample_surface(*room_mesh(0.1), 1000000, 0, None, 7, dev)
    rng = np.random.default_rng(0)
    K = 4096
    o = rng.uniform(-1, 1, size=(K, 3))
    cand = np.tile(np.eye(4), (K, 1, 1))
    cand[:, :3] = er.viewmatrix(rng.uniform(-1e4, 1e4, size=(K, 3)).round(2) - o, [0, 0, -1], o)
    ms = cuda_ms(lambda: er.points_seen(pts, cand, device=dev))
    rows.append(dict(what='unseen_check', candidates=K, points=pts.shape[0], ms=round(ms, 3)))
    print(json.dumps(rows[-1]), flush=True)
    # calc_2d_metric end to end: the 1 cm room against itself shifted by 1 cm, 1000 views
    gv, gf = room_mesh(0.01)
    with tempfile.TemporaryDirectory() as d:
        gt = io_formats.write_ply(os.path.join(d, 'room.ply'), gv, gf)
        rec = io_formats.write_ply(os.path.join(d, 'rec.ply'), gv + np.float32([0.01, 0, 0]), gf)
        a_ = np.stack(np.meshgrid(np.linspace(-1.5, 0.5, 100), np.linspace(-0.5, 1.5, 100)), -1)
        pc = np.concatenate([np.full((10000, 1), 2.9), a_.reshape(-1, 2)], 1).astype(np.float32)
        np.save(os.path.join(d, 'room_pc_unseen.npy'), pc)
        t0 = time.perf_counter()
        res = er.calc_2d_metric(rec, gt, align=False, n_imgs=1000, seed=0, device=dev)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
    rows.append(dict(what='calc_2d_metric', faces=len(gf), n_imgs=1000,
                     s=round(t1 - t0, 2), depth_l1_cm=round(res['depth l1'], 4)))
    print(json.dumps(rows[-1]), flush=True)
    # the numpy oracle, one 500 x 500 view of the 5 cm room
    v, f = room_mesh(0.05)
    w = np.linalg.inv(views(v, 1, 1))[:, :3]
    t0 = time.perf_counter()
    ore.render_depth(v, f, w, dict(H=500, W=500, fx=300., fy=300., cx=249.5, cy=249.5,
                                   near=0.063, far=20.))
    rows.append(dict(what='oracle_render', faces=len(f), s_per_view=round(time.perf_counter() - t0, 2)))
    print(json.dumps(rows[-1]), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, 'time_eval_2d.json'), 'w') as fh:
            json.dump(rows, fh, indent=1)


if __name__ == '__main__':
    main()
