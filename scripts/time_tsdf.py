"""Time Point-SLAM's TSDF mesh on the GPU: allocation, integration, extraction and clean_mesh
(csrc/tsdf.cu) for 10 and 40 keyframes of the synthetic 640x480 sequence, with CUDA events
after a warm-up, the block and (block, frame) pair counts, and the card / power limit.

    python scripts/time_tsdf.py [--out results/time_tsdf.json] [--frames 10 40] [--reps 3]

Needs a CUDA device; no fallback."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
                        '--format=csv,noheader'], capture_output=True, text=True).stdout
    return q.strip().splitlines()[0] if q.strip() else torch.cuda.get_device_name(0)


def run_once(dev, depth, color, c2w, w2c, intr):
    """One full pipeline with CUDA events between the phases -> (ms per phase, stats)."""
    from xrdslam_b200.tsdf import BLOCK_VOXELS, TSDFVolume, clean_mesh_arrays
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
    vol = TSDFVolume(device=dev)
    ev[0].record()
    keys, masks = vol.allocate(depth, torch.from_numpy(c2w[:, :3].copy()).to(dev), intr)
    ev[1].record()
    vol.integrate(depth, color, c2w, intr, w2c=w2c)   # allocates again: subtracted below
    ev[2].record()
    verts, faces, colors = vol.extract_triangle_mesh()
    ev[3].record()
    cv, cf, cc = clean_mesh_arrays(verts, faces, colors)
    ev[4].record()
    torch.cuda.synchronize()
    ms = [ev[i].elapsed_time(ev[i + 1]) for i in range(4)]
    bits = masks.cpu().numpy().view(np.uint32)
    pairs = int(sum(bin(int(x)).count('1') for x in bits.reshape(-1)))
    stats = {'blocks': int(keys.numel()), 'pairs': pairs,
             'voxel_frame_updates': pairs * BLOCK_VOXELS,
             'verts': int(verts.shape[0]), 'faces': int(faces.shape[0]),
             'clean_verts': int(cv.shape[0]), 'clean_faces': int(cf.shape[0])}
    return {'allocate': ms[0], 'integrate_incl_allocate': ms[1], 'extract': ms[2],
            'clean': ms[3]}, stats


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--frames', type=int, nargs='+', default=[10, 40])
    ap.add_argument('--reps', type=int, default=3)
    a = ap.parse_args()
    from xrdslam_b200.synthetic import make_sequence
    from xrdslam_b200.tsdf import o3d_poses
    dev = torch.device('cuda:0')
    res = {'card': card(), 'runs': []}
    print(res['card'])
    for K in a.frames:
        cam, poses, frames = make_sequence(K)
        c2w, w2c = o3d_poses(poses)
        depth = torch.from_numpy(np.stack([d for _, d in frames])).to(dev)
        color = torch.from_numpy(np.stack([(rgb * 255).astype(np.uint8) for rgb, _ in frames])).to(dev)
        intr = (cam.fx, cam.fy, cam.cx, cam.cy)
        run_once(dev, depth, color, c2w, w2c, intr)   # warm-up
        best = None
        for _ in range(a.reps):
            ms, stats = run_once(dev, depth, color, c2w, w2c, intr)
            best = ms if best is None else {k: min(best[k], ms[k]) for k in ms}
        best['integrate'] = best['integrate_incl_allocate'] - best['allocate']
        rate = stats['voxel_frame_updates'] / (best['integrate'] * 1e-3)
        r = {'keyframes': K, 'size': [cam.width, cam.height], 'ms_best_of_reps': best,
             'voxel_frame_updates_per_s': rate, **stats}
        print(json.dumps(r))
        res['runs'].append(r)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as fh:
            json.dump(res, fh, indent=1)


if __name__ == '__main__':
    main()
