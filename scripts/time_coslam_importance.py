"""Co-SLAM with importance sampling (training_n_importance = N): the 4096-ray mapping iteration
(graph session: coarse pass, importance step, fine pass, smoothness, Adam) and a 1024-ray
tracking iteration, at N in {0, 16, 48}, each on the tile kernel (rays_per_tile = -1) and with the
automatic kernel choice (rays_per_tile = 0), in alternating rounds in one process.  Prints the GPU
name, power limit and SM clocks with the medians.
    python scripts/time_coslam_importance.py [--iters 50] [--rounds 5]"""
import argparse
import os
import random
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import bench  # noqa: E402

CONFIGS = {f'N = {n}, {name}': dict(n_importance=n, rays_per_tile=rpt)
           for n in (0, 16, 48) for name, rpt in (('tile kernel', -1), ('automatic', 0))}


def build(dev, seed, n_importance, rays_per_tile):
    from xrdslam_b200.coslam import CoSLAMConfig
    from xrdslam_b200.frame import Frame
    from xrdslam_b200.synthetic import make_sequence
    random.seed(seed)
    np.random.seed(seed)
    torch.manual_seed(seed)
    cam, poses, frames = make_sequence(bench.N_KEYFRAMES + 1)
    cfg = CoSLAMConfig()
    cfg.model.precision = 1
    cfg.model.training_n_importance = n_importance
    cfg.model.rays_per_tile = rays_per_tile
    algo = cfg.setup(camera=cam, device=dev)
    kfs = []
    for k in range(bench.N_KEYFRAMES):
        f = Frame(k, frames[k][0], frames[k][1], init_pose=poses[k], separate_LR=True,
                  rot_rep='axis_angle')
        algo.add_keyframe(f)
        kfs.append(f)
    cur = Frame(bench.N_KEYFRAMES, frames[-1][0], frames[-1][1], init_pose=poses[-1],
                separate_LR=True, rot_rep='axis_angle')
    algo.set_initialized()
    frames = kfs + [cur]
    algo.config.mapping_sample = bench.MAP_KF
    algo.config.min_sample_pixels = bench.MAP_CUR
    algo.config.tracking_sample = 1024
    algo.bundle_adjust = True
    algo.setup_optimizers(1000, frames, is_mapping=True)
    sess = algo.mapping_session(frames)
    sess.begin(frames)
    batch = sess.make_resident_batch(frames)
    trk = algo.tracking_session()
    trk.begin(cur)
    return sess, batch, trk


def timed(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for i in range(iters):
        fn(i)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--rounds', type=int, default=5)
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm',
                        '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip()
    print('GPU:', q or torch.cuda.get_device_name(dev))
    runs = {k: build(dev, 1234, **c) for k, c in CONFIGS.items()}
    for sess, batch, trk in runs.values():  # warm-up
        for i in range(5):
            sess.step_resident(i, batch)
            trk.step()
    res = {k: ([], []) for k in runs}
    for _ in range(args.rounds):
        for k, (sess, batch, trk) in runs.items():
            res[k][0].append(timed(lambda i: sess.step_resident(i, batch), args.iters))
            res[k][1].append(timed(lambda i: trk.step(), args.iters))
    print(f'{"configuration":24s} {"mapping 4096 rays (ms)":>24s} {"tracking 1024 rays (ms)":>24s}')
    q = subprocess.run(['nvidia-smi', '--query-gpu=clocks.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip()
    print('SM clock after the rounds:', q)
    for k, (m, t) in res.items():
        print(f'{k:24s} {np.median(m):24.3f} {np.median(t):24.3f}   '
              f'(spread {min(m):.3f}-{max(m):.3f} / {min(t):.3f}-{max(t):.3f})')


if __name__ == '__main__':
    main()
