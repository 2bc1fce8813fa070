"""Time mesh extraction on the GPU: get_mesh for Co-SLAM and NICE-SLAM at resolution 256 and
Vox-Fusion extract_mesh on a map grown from synthetic 640x480 frames, with per-phase CUDA-event
times (query, marching cubes, colour) and the CPU oracle's time for the same pipeline.

    python scripts/time_mesh.py [--out results/time_mesh.json] [--cpu-res 64]

Models carry seeded random parameters scaled so that a surface exists (the timings depend on
the lattice size and the mesh size, which are printed).  Needs a CUDA device; no fallback."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
                        '--format=csv,noheader'], capture_output=True, text=True).stdout
    return q.strip().splitlines()[0] if q.strip() else torch.cuda.get_device_name(0)


class Phases:
    def __init__(self):
        self.ev = []

    def mark(self, name):
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        self.ev.append((name, e))

    def ms(self):
        torch.cuda.synchronize()
        return {self.ev[i + 1][0]: round(self.ev[i][1].elapsed_time(self.ev[i + 1][1]), 3)
                for i in range(len(self.ev) - 1)}


def time_mesher(algo, reps=2):
    """Wall time of get_mesh (best of reps, after one warm-up) and one phase-timed run."""
    algo.get_mesh()
    walls = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t = time.perf_counter()
        mesh = algo.get_mesh()
        torch.cuda.synchronize()
        walls.append(time.perf_counter() - t)
    m, dev = algo.mesher, algo.device
    p = Phases()
    with torch.no_grad():
        p.mark('start')
        vol, xyz = m.query_volume(algo.model.query_fn, dev)
        p.mark('query')
        verts, faces = m.extract(vol, xyz)
        p.mark('marching_cubes')
        m.vertex_colors(verts, algo.model.color_func, dev)
        p.mark('colour')
    return dict(wall_s=round(min(walls), 4), phases_ms=p.ms(), lattice=list(vol.shape[1:]),
                verts=int(mesh.vertices.shape[0]), faces=int(mesh.faces.shape[0])), vol


def coslam(dev):
    from oracle.coslam import CoslamOracle
    from xrdslam_b200.coslam import CoSLAMConfig
    from xrdslam_b200.synthetic import make_camera
    cfg = CoSLAMConfig()
    algo = cfg.setup(camera=make_camera(640, 480), device=dev)
    ora = CoslamOracle(np.array(cfg.mapping_bound, dtype=np.float64))
    g = torch.Generator().manual_seed(1)
    with torch.no_grad():
        ora.embed_fn.params.copy_((torch.rand(ora.embed_fn.params.shape, generator=g) * 2 - 1) * 0.3)
        for lin in (ora.sdf0, ora.sdf1, ora.col0, ora.col1):
            lin.weight.copy_(torch.randn(lin.weight.shape, generator=g) / np.sqrt(lin.weight.shape[1]))
        m = algo.model
        m.embed_fn.params.copy_(ora.embed_fn.params)
        m.decoder.sdf_net.model[0].weight.copy_(ora.sdf0.weight)
        m.decoder.sdf_net.model[2].weight.copy_(ora.sdf1.weight)
        m.decoder.color_net.model[0].weight.copy_(ora.col0.weight)
        m.decoder.color_net.model[2].weight.copy_(ora.col1.weight)
    return algo, ora


def coslam_cpu(algo, ora, res):
    """The same pipeline on the CPU oracle at resolution `res`: float64 queries, numpy marching
    cubes, colour queries."""
    from oracle.marching_cubes import marching_cubes
    from xrdslam_b200.mesher import Mesher, MesherConfig
    m = Mesher(MesherConfig(resolution=res), None, algo.bounding_box, algo.marching_cube_bound)
    bb = torch.as_tensor(algo.bounding_box, dtype=torch.float64)
    q = lambda p: ora.query_color_sdf((p.double() - bb[:, 0]) / (bb[:, 1] - bb[:, 0]))
    t = {}
    with torch.no_grad():
        t0 = time.perf_counter()
        xyz = m.get_grid_uniform(res)['xyz']
        pts = m.grid_points(xyz, 0, res ** 3, 'cpu')
        vol = m.eval_points(pts, lambda p: q(p)[:, 3:4].float(), m.bounding_box, 'cpu')[:, -1]
        t['query'] = time.perf_counter() - t0
        t0 = time.perf_counter()
        v, f = marching_cubes(vol.numpy().reshape(1, res, res, res), 0.0,
                              [a[2] - a[1] for a in xyz], [a[0] for a in xyz])
        t['marching_cubes'] = time.perf_counter() - t0
        t0 = time.perf_counter()
        m.eval_points(torch.from_numpy(v), lambda p: torch.sigmoid(q(p)[:, :3]).float(),
                      m.bounding_box, 'cpu')
        t['colour'] = time.perf_counter() - t0
    return dict(resolution=res, phases_s={k: round(x, 3) for k, x in t.items()},
                total_s=round(sum(t.values()), 3), faces=int(f.shape[0]))


def nice(dev):
    import warnings
    from xrdslam_b200.nice_slam import NiceSLAMConfig
    from xrdslam_b200.synthetic import make_camera
    torch.manual_seed(0)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        algo = NiceSLAMConfig().setup(camera=make_camera(640, 480), device=dev)
    with torch.no_grad():
        for g in algo.model.grids.values():
            g.mul_(30.0)
    return algo


def voxfusion(dev, n_frames=3):
    from xrdslam_b200.synthetic import make_sequence
    from xrdslam_b200.voxfusion import VoxFusionConfig
    cam, poses, frames = make_sequence(n_frames, width=640, height=480, offset=(25.6,) * 3)
    torch.manual_seed(0)
    algo = VoxFusionConfig().setup(camera=cam, device=dev)
    H, W = cam.height, cam.width
    j, i = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32),
                          indexing='ij')
    dirs = torch.stack([(i - cam.cx) / cam.fx, -(j - cam.cy) / cam.fy, -torch.ones_like(i)], -1)
    for (rgb, depth), c2w in zip(frames, poses):
        c2w, d = torch.from_numpy(c2w), torch.from_numpy(depth)
        pts = (dirs * d[..., None])[d > 0].reshape(-1, 3)
        algo.model.insert_points((pts @ c2w[:3, :3].T + c2w[:3, 3]).to(dev))
    g = torch.Generator().manual_seed(1)
    with torch.no_grad():
        algo.model.embeddings.copy_(torch.randn(algo.model.embeddings.shape, generator=g))
        ids, _, _ = algo.surface_voxels()
        algo.model.decoder.sdf_out.bias[0] -= algo.model.get_scores(ids, 4).median()
    return algo


def time_vox(algo, reps=2):
    from xrdslam_b200.mesher import marching_cubes
    algo.get_mesh()
    walls = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t = time.perf_counter()
        mesh = algo.get_mesh()
        torch.cuda.synchronize()
        walls.append(time.perf_counter() - t)
    vs = algo.model.config.voxel_size
    p = Phases()
    with torch.no_grad():
        p.mark('start')
        ids, voxels, centres = algo.surface_voxels()
        sdf = algo.model.get_scores(ids, 8)
        p.mark('query')
        verts, faces = marching_cubes(sdf, 0.0, (1 / 7,) * 3, (-0.5,) * 3, (vs,) * 3, centres)
        p.mark('marching_cubes')
        algo.vertex_colors(verts, ids, voxels)
        p.mark('colour')
    return dict(wall_s=round(min(walls), 4), phases_ms=p.ms(), surface_voxels=int(ids.numel()),
                verts=int(mesh.vertices.shape[0]), faces=int(mesh.faces.shape[0])), sdf, centres


def vox_cpu_mc(sdf, centres, vs):
    """numpy marching cubes of the same batched volume (the CPU restatement of the kernels)."""
    from oracle.marching_cubes import marching_cubes
    s, c = sdf.cpu().numpy(), centres.cpu().numpy()
    t0 = time.perf_counter()
    marching_cubes(s, 0.0, (1 / 7,) * 3, (-0.5,) * 3, (vs,) * 3, c)
    return round(time.perf_counter() - t0, 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--cpu-res', type=int, default=64)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('time_mesh.py needs a CUDA device')
    from xrdslam_b200 import _cabi
    _cabi.check('xrd_check_device', _cabi.lib().xrd_check_device(0))
    dev = torch.device('cuda:0')
    res = {'card': card(), 'torch': torch.__version__}
    algo, ora = coslam(dev)
    res['coslam'], vol = time_mesher(algo)
    from oracle.marching_cubes import marching_cubes
    xyz = algo.mesher.get_grid_uniform(algo.mesher.config.resolution)['xyz']
    t0 = time.perf_counter()
    marching_cubes(vol.cpu().numpy(), 0.0, [x[2] - x[1] for x in xyz], [x[0] for x in xyz])
    res['coslam']['cpu_oracle_mc_same_volume_s'] = round(time.perf_counter() - t0, 3)
    res['coslam']['cpu_oracle_pipeline'] = coslam_cpu(algo, ora, a.cpu_res)
    del algo, ora, vol
    torch.cuda.empty_cache()
    algo = nice(dev)
    res['nice'], vol = time_mesher(algo)
    del algo, vol
    torch.cuda.empty_cache()
    algo = voxfusion(dev)
    res['voxfusion'], sdf, centres = time_vox(algo)
    res['voxfusion']['cpu_oracle_mc_same_volume_s'] = vox_cpu_mc(sdf, centres, algo.model.config.voxel_size)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
