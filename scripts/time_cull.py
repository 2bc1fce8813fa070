"""Time cull_mesh on the GPU (csrc/cull.cu, common.cull_mesh): seeded vertices in and around the
synthetic room, n frames at 640x480 and 1200x680 with host depth; per-phase CUDA-event times
(upload = host staging + H2D + the per-frame torch.inverse; visibility = the kernel launches;
compaction = count + emit), whole-call wall time, and the vertex-frame tests the kernel
actually executes (it stops at a vertex's first seeing frame, so fewer than the nominal V * n)
per second of kernel time.  A second workload puts every vertex behind a wall, so no vertex is
ever seen and all V * n tests run.  Leg (b) -- the reference's
per-frame torch loop restated in oracle/cull.py, on the same GPU, same inputs -- is timed beside
it, and its decisions are compared.  The card and its power limit are read in the same call.

    python scripts/time_cull.py [--out results/time_cull.json] [--verts 1000000 4500000]
                                [--frames 2000] [--ref-frames 200]

Leg (b) runs the first --ref-frames frames; the speed-up is measured against cull_visibility on
those same frames.  Needs a CUDA device; no fallback."""
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


class SynthDataset:
    """n frames cycling over 16 rendered views of the synthetic room (host depth tensors)."""

    def __init__(self, n, width, height, n_views=16):
        from xrdslam_b200.synthetic import make_sequence
        self.cam, poses, frames = make_sequence(n_views, width=width, height=height)
        self.poses = [torch.from_numpy(p) for p in poses]
        self.depth = [torch.from_numpy(d) for _, d in frames]
        self.n = n

    def __len__(self):
        return self.n

    def __getitem__(self, i):
        k = i % len(self.depth)
        return i, None, self.depth[k], self.poses[k]

    def get_camera(self):
        return self.cam


def vertices(V, seed=0):
    from xrdslam_b200.synthetic import ROOM
    rng = np.random.default_rng(seed)
    v = rng.uniform(ROOM[:, 0] - 0.3, ROOM[:, 1] + 0.3, (V, 3)).astype(np.float32)
    f = rng.integers(0, V, (2 * V, 3)).astype(np.int32)
    return v, f


def occluded_vertices(V, seed=1):
    """Vertices 0.5-1.5 m outside the room's walls: every frame that projects one into its image
    has a wall more than the truncation in front of it, so no vertex is ever seen and the kernel
    executes all V * n tests."""
    from xrdslam_b200.synthetic import ROOM
    rng = np.random.default_rng(seed)
    out = []
    while sum(len(o) for o in out) < V:
        p = rng.uniform(ROOM[:, 0] - 1.5, ROOM[:, 1] + 1.5, (V, 3))
        out.append(p[((p < ROOM[:, 0] - 0.5) | (p > ROOM[:, 1] + 0.5)).any(1)])
    v = np.concatenate(out)[:V].astype(np.float32)
    f = rng.integers(0, V, (2 * V, 3)).astype(np.int32)
    return v, f


def _resident(dev, ds):
    from xrdslam_b200.common import cull_w2c
    depth = torch.stack([d for d in ds.depth]).to(dev)
    w2c = torch.stack([cull_w2c(p.to(dev)) for p in ds.poses]).contiguous()
    return depth, w2c


def executed_tests(dev, ds, verts_d):
    """Vertex-frame tests the kernel executes: a vertex is tested in frame f iff no earlier frame
    saw it (the early exit inside a launch and the skip at a launch's start give the same count
    for any chunking).  Replayed one frame per launch, counting the unseen vertices first."""
    import ctypes as C
    from xrdslam_b200 import _cabi
    cam = ds.get_camera()
    depth, w2c = _resident(dev, ds)
    P = _cabi.XrdCullParams(cam.height, cam.width, cam.fx, cam.fy, cam.cx, cam.cy, 0.06, 1)
    seen = torch.zeros(verts_d.shape[0], dtype=torch.uint8, device=dev)
    total = torch.zeros((), dtype=torch.int64, device=dev)
    lib = _cabi.lib()
    s = torch.cuda.current_stream(dev).cuda_stream
    for f in range(len(ds)):
        total += (seen == 0).sum()
        k = f % len(ds.depth)
        _cabi.check('xrd_cull_visible', lib.xrd_cull_visible(
            _cabi.ptr(verts_d), verts_d.shape[0], _cabi.ptr(w2c[k]), _cabi.ptr(depth[k]), 1,
            C.byref(P), _cabi.ptr(seen), s))
    return int(total)


def run_cull(dev, ds, verts_d, faces_d, chunk):
    """-> (ms per phase, wall s, seen, (V', F'))."""
    from xrdslam_b200 import common
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ev[0].record()
    seen = common.cull_visibility(ds, verts_d, None, True, 0.06, dev, chunk)
    ev[1].record()
    v, f, _ = common.cull_compact(seen, verts_d, faces_d)
    ev[2].record()
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    return ({'visibility_incl_upload': ev[0].elapsed_time(ev[1]),
             'compaction': ev[1].elapsed_time(ev[2])}, wall, seen, (v.shape[0], f.shape[0]))


def kernel_only(dev, ds, verts_d, chunk):
    """The visibility launches alone over device-resident chunks: -> ms."""
    import ctypes as C
    from xrdslam_b200 import _cabi
    cam = ds.get_camera()
    H, W = cam.height, cam.width
    n = len(ds)
    views = len(ds.depth)
    depth, w2c = _resident(dev, ds)
    P = _cabi.XrdCullParams(H, W, cam.fx, cam.fy, cam.cx, cam.cy, 0.06, 1)
    seen = torch.zeros(verts_d.shape[0], dtype=torch.uint8, device=dev)
    lib = _cabi.lib()
    s = torch.cuda.current_stream(dev).cuda_stream
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for k in range(0, n, chunk):
        m = min(chunk, n - k)
        # chunks of views 0..m-1 (visibility is an OR, so repeating views costs the same tests)
        assert m <= views
        _cabi.check('xrd_cull_visible', lib.xrd_cull_visible(
            _cabi.ptr(verts_d), verts_d.shape[0], _cabi.ptr(w2c), _cabi.ptr(depth), m,
            C.byref(P), _cabi.ptr(seen), s))
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def run_reference(dev, ds, verts, n):
    from oracle.cull import reference_seen
    sub = SynthDataset.__new__(SynthDataset)
    sub.__dict__.update(ds.__dict__)
    sub.n = n
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    seen = reference_seen(sub, verts, None, True, 0.06, device=dev)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, seen


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--verts', type=int, nargs='+', default=[1000000, 4500000])
    ap.add_argument('--frames', type=int, default=2000)
    ap.add_argument('--ref-frames', type=int, default=200)
    ap.add_argument('--chunk', type=int, default=16)
    a = ap.parse_args()
    from xrdslam_b200.common import cull_visibility
    dev = torch.device('cuda:0')
    res = {'card': card(), 'runs': []}
    print(res['card'], flush=True)
    for (w, h) in ((640, 480), (1200, 680)):
        ds = SynthDataset(a.frames, w, h)
        for V, workload in [(V, w) for V in a.verts for w in ('random', 'occluded')]:
            verts, faces = (vertices if workload == 'random' else occluded_vertices)(V)
            vd, fd = torch.from_numpy(verts).to(dev), torch.from_numpy(faces).to(dev)
            warm = SynthDataset.__new__(SynthDataset)
            warm.__dict__.update(ds.__dict__)
            warm.n = 2 * a.chunk
            run_cull(dev, warm, vd, fd, a.chunk)                      # warm-up
            ms, wall, seen, counts = run_cull(dev, ds, vd, fd, a.chunk)
            kms = kernel_only(dev, ds, vd, a.chunk)
            tests = V * a.frames
            executed = executed_tests(dev, ds, vd)
            r = {'size': [w, h], 'workload': workload, 'verts': V, 'faces': 2 * V,
                 'frames': a.frames, 'chunk': a.chunk,
                 'ms': {**ms, 'visibility_kernels_device_resident': kms,
                        'upload_and_inverse': ms['visibility_incl_upload'] - kms},
                 'wall_s': wall, 'seen': int(seen.sum()), 'kept_V_F': list(counts),
                 'vertex_frame_tests_nominal': tests, 'vertex_frame_tests_executed': executed,
                 'executed_tests_per_s_kernels': executed / (kms * 1e-3)}
            if workload == 'occluded':
                print(json.dumps(r), flush=True)
                res['runs'].append(r)
                continue
            nref = min(a.ref_frames, a.frames)
            run_reference(dev, warm, verts, 2)                        # warm-up
            ref_s, ref_seen = run_reference(dev, ds, verts, nref)
            # decisions of the first nref frames, for the comparison
            part = SynthDataset.__new__(SynthDataset)
            part.__dict__.update(ds.__dict__)
            part.n = nref
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            seen_n = cull_visibility(part, vd, None, True, 0.06, dev, a.chunk)
            torch.cuda.synchronize()
            ours_s = time.perf_counter() - t0
            diff = int((seen_n.bool() != ref_seen).sum())
            r['reference_leg_b'] = {'frames': nref, 's': ref_s, 's_per_frame': ref_s / nref,
                                    'seen_disagreements': diff,
                                    'cull_visibility_s_same_frames': ours_s,
                                    'speedup_same_frames': ref_s / ours_s}
            print(json.dumps(r), flush=True)
            res['runs'].append(r)
            del vd, fd
            torch.cuda.empty_cache()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as fh:
            json.dump(res, fh, indent=1)


if __name__ == '__main__':
    main()
