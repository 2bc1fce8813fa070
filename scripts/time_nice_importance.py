"""NICE-SLAM with stratified jitter and importance sampling: ms per fused mapping iteration
(stage colour, 5000 rays, colour decoder trained) and tracking iteration (200 rays, ray
gradients only) at n_importance in {0, 16, 80}, rendering_perturb 0 and 1, in alternating rounds
in one process.  Reports ms and rays/s, with the GPU name and power limit read in the same run.
    python scripts/time_nice_importance.py [--iters 30] [--rounds 3]"""
import argparse
import os
import subprocess
import sys
import warnings

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

BOUND = np.array([[-3.2, 3.2], [-4.2, 2.7], [-2.2, 2.7]])


def model(dev, n, perturb):
    from xrdslam_b200.camera import Camera
    from xrdslam_b200.conv_onet import ConvOnetConfig
    with warnings.catch_warnings():
        warnings.simplefilter('ignore', RuntimeWarning)
        m = ConvOnetConfig(rendering_n_importance=n, rendering_perturb=perturb,
                           mapping_frustum_feature_selection=False).setup(
            camera=Camera(320., 320., 319.5, 239.5, 640, 480), bounding_box=BOUND)
    return m.to(dev)


def batch(dev, R, seed):
    g = torch.Generator().manual_seed(seed)
    ro = torch.rand(R, 3, generator=g) * 0.5
    rd = torch.nn.functional.normalize(torch.randn(R, 3, generator=g), dim=-1)
    td = torch.rand(R, 1, generator=g) * 3 + 0.3
    ts = torch.rand(R, 3, generator=g)
    return [t.to(dev) for t in (ro, rd, ts, td)]


def time_it(m, dev, is_mapping, R, iters):
    ro, rd, ts, td = batch(dev, R, R)
    args = ('color', is_mapping, ro, rd, ts, td, True)
    kw = dict(need_rays=not is_mapping, need_grid=(is_mapping,) * 3, need_col=is_mapping)
    for _ in range(3):
        m._launch(*args, **kw)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        m._launch(*args, **kw)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=30)
    ap.add_argument('--rounds', type=int, default=3)
    a = ap.parse_args()
    dev = torch.device('cuda:0')
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip()
    print('GPU:', torch.cuda.get_device_name(dev), '|', q)
    cfgs = [(n, p) for n in (0, 16, 80) for p in (0.0, 1.0)]
    models = {c: model(dev, *c) for c in cfgs}
    res = {(c, k): [] for c in cfgs for k in ('map', 'trk')}
    for _ in range(a.rounds):
        for c in cfgs:
            res[(c, 'map')].append(time_it(models[c], dev, True, 5000, a.iters))
            res[(c, 'trk')].append(time_it(models[c], dev, False, 200, a.iters))
    for c in cfgs:
        for k, R in (('map', 5000), ('trk', 200)):
            ms = float(np.median(res[(c, k)]))
            print(f'N = {c[0]:2d}, perturb = {c[1]:.0f}, {k}: {ms:.3f} ms/iter, '
                  f'{R / ms * 1e3:.4g} rays/s')


if __name__ == '__main__':
    main()
