"""Time the Co-SLAM fused pass on random rays (tests/helpers.py).

  quick_time_coslam.py [NR ...]
      fwd+bwd and forward-only per call of Model._launch at R = 1024 .. 65536, for each
      rays_per_tile value NR (0 auto, -1 tile kernel, -2 grouped kernel).
  quick_time_coslam.py --passes [NR ...]
      the fused kernel alone (CUDA events the library records around its launch, L2 flushed
      before every launch) at --rays rays for three passes:
        fwd   forward only
        pose  + the corner re-gather for d loss / d x and the ray gradients
        full  + the table-gradient scatter and the weight gradients (mapping with bundle
              adjustment, the benchmark's pass)
XRD_PREC selects cfg.precision (default 0; the benchmark runs 1).
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
import numpy as np
import torch
from helpers import coslam_pair, make_rays
from xrdslam_b200 import _cabi

ap = argparse.ArgumentParser()
ap.add_argument('nr', nargs='*', type=int, default=[0])
ap.add_argument('--passes', action='store_true')
ap.add_argument('--rays', type=int, default=4096)
ap.add_argument('--iters', type=int, default=50)
args = ap.parse_args()

dev = torch.device('cuda:0')
_, model = coslam_pair(dev, table_amp=1e-2, precision=int(os.environ.get("XRD_PREC", "0")))
w = model._weights()
tab = model.embed_fn.params


def rays(R):
    rays_o, rays_d, ts, td, _ = make_rays(R, seed=1)
    return [t.to(dev) for t in (rays_o, rays_d, ts, td)]


def run(inp, grads=True, map_grads=True):
    ro, rd, ts, td = inp
    return model._launch(ro, rd, tab, *w, ts, td, None, with_grads=grads, map_grads=map_grads)


PASSES = {'fwd': dict(grads=False), 'pose': dict(grads=True, map_grads=False),
          'full': dict(grads=True, map_grads=True)}

if args.passes:
    lib = _cabi.lib()
    flush = torch.empty(64 << 20, dtype=torch.float32, device=dev)  # 256 MB > 50 MB L2
    inp = rays(args.rays)
    print(f'{torch.cuda.get_device_name(dev)}, R={args.rays}, precision {model.config.precision}; '
          f'fused kernel median / mean over {args.iters} launches, us')
    for nr in args.nr:
        model.config.rays_per_tile = nr
        row = []
        for name, kw in PASSES.items():
            for _ in range(3):
                run(inp, **kw)
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
                  for _ in range(args.iters)]
            for a, b in ev:
                flush.zero_()
                a.record()  # materialise the handles; the library re-records both
                b.record()
                lib.xrd_debug_kernel_events(a.cuda_event, b.cuda_event)
                run(inp, **kw)
                lib.xrd_debug_kernel_events(None, None)
            torch.cuda.synchronize()
            t = np.array([a.elapsed_time(b) for a, b in ev]) * 1e3
            row.append(f'{name} {np.median(t):7.1f} / {t.mean():7.1f}')
        print(f'NR={nr}: ' + '   '.join(row))
    sys.exit(0)

for R in [1024, 4096, 16384, 65536]:
    inp = rays(R)
    for nr in args.nr:
        model.config.rays_per_tile = nr  # 0 auto, -1 tile kernel, -2 grouped kernel
        for _ in range(3): run(inp)
        torch.cuda.synchronize()
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        n = 20
        e0.record()
        for _ in range(n): run(inp)
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / n
        e0.record()
        for _ in range(n): run(inp, False)
        e1.record(); torch.cuda.synchronize()
        msf = e0.elapsed_time(e1) / n
        print(f'R={R} NR={nr}: fwd+bwd {ms*1e3:.1f} us  ({R/ms/1e3:.2f} Mrays/s, {R*88064/ms/1e6:.1f} GB/s algorithmic)   fwd-only {msf*1e3:.1f} us')
