"""Time the render-quality metrics on the device (csrc/eval_image.cu).

Reports, with the card name, power limit and SM clocks: xrd_eval_image_metrics for B = 1 and
B = 40 frames of 640 x 480 (best of N, CUDA events); the reference's torch metric code (oracle
(b): F.mse_loss, pytorch_msssim.ms_ssim restated, the masked depth L1) on the same GPU, one frame
per call as save_render_imgs runs it; and Algorithm.eval_re_render per algorithm on a synthetic
640 x 480 sequence, split into render_img(to_host=False) and metrics time per frame.  Prints one
JSON line per measurement and, with --out, writes them all to <out>/time_eval_image.json.

    python scripts/time_eval_image.py [--out DIR] [--reps N]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from oracle import eval_image as oe  # noqa: E402
from xrdslam_b200.eval_image import image_metrics  # noqa: E402
from xrdslam_b200.synthetic import make_sequence  # noqa: E402


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


def reference_metrics(gc, gd, c, d):
    """The torch part of save_render_imgs on device tensors of one frame (oracle (b))."""
    gc, c = gc.clamp(0, 1), c.clamp(0, 1)
    ok = gd > 0
    dl1 = torch.abs(gd[ok] - d[ok]).mean() * 100
    psnr = -10. * torch.log10(F.mse_loss(gc, c))
    ssim = oe.ms_ssim(gc.transpose(0, 2).unsqueeze(0), c.transpose(0, 2).unsqueeze(0),
                      data_range=1.0)
    return psnr, ssim, dl1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--reps', type=int, default=20)
    a = ap.parse_args()
    dev = torch.device('cuda:0')
    rows = [dict(card=card())]

    def emit(**kw):
        rows.append(kw)
        print(json.dumps(kw), flush=True)

    _, _, fr = make_sequence(41)
    t = lambda x, dt: torch.from_numpy(np.stack(x)).to(dev, dt)
    gc = t([f[0] for f in fr[:40]], torch.float32)
    gd = t([f[1] for f in fr[:40]], torch.float32)
    c = t([f[0] for f in fr[1:]], torch.float32)
    d = t([f[1] for f in fr[1:]], torch.float64)
    for B in (1, 40):
        out = torch.empty(B, 4, dtype=torch.float64, device=dev)
        ms = cuda_ms(lambda: image_metrics(gc[:B], gd[:B], c[:B], d[:B], out=out), a.reps)
        emit(what='metrics', B=B, H=480, W=640, ms=round(ms, 4), ms_per_frame=round(ms / B, 4))
    ms = cuda_ms(lambda: [reference_metrics(gc[k], gd[k], c[k], d[k]) for k in range(40)],
                 max(1, a.reps // 4))
    emit(what='reference_torch_metrics', B=40, H=480, W=640, ms_per_frame=round(ms / 40, 4))

    from test_eval_image_gpu import _algorithm
    n = 4
    for name in ('coslam', 'nice', 'voxfusion', 'pointslam'):
        algo, ds = _algorithm(name, dev, width=640, height=480, n_frames=n)
        algo.eval_re_render(ds, render_freq=1, estimate_c2w_list=ds.poses)   # warm-up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        algo.eval_re_render(ds, render_freq=1, estimate_c2w_list=ds.poses)
        torch.cuda.synchronize()
        wall = (time.perf_counter() - t0) * 1e3 / n
        render, metric = [], []
        for i in range(n):
            _, rgb, depth, c2w = ds[i]
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
            ev[0].record()
            col, dep = algo.render_img(c2w, gt_depth=depth, idx=i, to_host=False)
            ev[1].record()
            image_metrics(torch.from_numpy(rgb).to(dev)[None], torch.from_numpy(depth).to(dev)[None],
                          col[None], dep[None])
            ev[2].record()
            ev[2].synchronize()
            render.append(ev[0].elapsed_time(ev[1]))
            metric.append(ev[1].elapsed_time(ev[2]))
        emit(what='eval_re_render', algorithm=name, H=480, W=640, frames=n,
             wall_ms_per_frame=round(wall, 2), render_ms_per_frame=round(float(np.median(render)), 2),
             metrics_ms_per_frame=round(float(np.median(metric)), 3))
        del algo, ds
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, 'time_eval_image.json'), 'w') as fh:
            json.dump(rows, fh, indent=1)


if __name__ == '__main__':
    main()
