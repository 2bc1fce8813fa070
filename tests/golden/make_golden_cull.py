"""Write tests/golden/cull_mesh_ref.npz: the reference's own cull_mesh (slam/common/common.py:
714-789) run on CPU through oracle/ref_harness.py on seeded inputs, so that the GPU tests (where
the reference is absent) meet its decisions.

    python tests/golden/make_golden_cull.py

A stub mesh records the face mask cull_mesh passes to update_faces.  One degenerate face
(v, v, v) per vertex is appended to the real faces, so the same mask also holds whole_mask:
~whole_mask[v] is the kept flag of face F + v.  Stored per case: seen (= ~whole_mask) and the
kept-face mask of the real faces, with the inputs (vertices, faces, depth, dataset poses,
estimate poses, camera)."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

# (name, use estimate_c2w_list, eval_rec, truncation)
CASES = [('est_rec', True, True, 0.06), ('ds_norec', False, False, 0.06),
         ('ds_rec_t02', False, True, 0.02)]


def inputs(n_frames=5, width=160, height=120, n_surface=4000, n_box=2000, n_faces=8000, seed=0):
    """Seeded vertices near the synthetic room's surfaces (back-projected depth + noise) and in
    and around its box, random faces over them, and estimate poses for all but the last frame."""
    from xrdslam_b200.synthetic import ROOM, make_sequence
    rng = np.random.default_rng(seed)
    cam, poses, frames = make_sequence(n_frames, width, height)
    depth = np.stack([d for _, d in frames]).astype(np.float32)
    pts = []
    for k in range(n_frames):
        r, c = rng.integers(0, height, n_surface // n_frames), rng.integers(0, width, n_surface // n_frames)
        d = depth[k, r, c].astype(np.float64)
        cam_p = np.stack([(c - cam.cx) / cam.fx * d, -(r - cam.cy) / cam.fy * d, -d], -1)
        pts.append(cam_p @ poses[k][:3, :3].T.astype(np.float64) + poses[k][:3, 3])
    surf = np.concatenate(pts) + rng.normal(0, 0.05, (n_surface // n_frames * n_frames, 3))
    box = rng.uniform(ROOM[:, 0] - 0.5, ROOM[:, 1] + 0.5, (n_box, 3))
    verts = np.concatenate([surf, box]).astype(np.float32)
    faces = rng.integers(0, verts.shape[0], (n_faces, 3)).astype(np.int32)
    est = np.stack(poses[:-1]).astype(np.float32)
    est[:, :3, 3] += rng.normal(0, 0.01, (n_frames - 1, 3)).astype(np.float32)
    cam_arr = np.array([cam.height, cam.width, cam.fx, cam.fy, cam.cx, cam.cy], np.float64)
    return dict(verts=verts, faces=faces, depth=depth, poses=np.stack(poses).astype(np.float32),
                est=est, camera=cam_arr)


class Dataset:
    """The three things cull_mesh reads from a dataset: len, [i] -> (idx, rgb, depth, c2w),
    get_camera()."""

    def __init__(self, depth, poses, camera, device='cpu'):
        from xrdslam_b200.camera import Camera
        h, w, fx, fy, cx, cy = camera
        self.cam = Camera(fx, fy, cx, cy, int(w), int(h))
        self.depth = torch.as_tensor(depth).to(device)
        self.poses = torch.as_tensor(poses).to(device)

    def __len__(self):
        return self.depth.shape[0]

    def __getitem__(self, i):
        return i, None, self.depth[i], self.poses[i]

    def get_camera(self):
        return self.cam


class _RecordingMesh:
    def __init__(self, vertices, faces):
        self.vertices, self.faces = vertices, faces

    def update_faces(self, mask):
        self.kept = np.asarray(mask).copy()

    def remove_unreferenced_vertices(self):
        pass

    def process(self, validate=False):
        pass


def reference_decisions(inp, use_est, eval_rec, truncation):
    """-> (seen bool [V], kept bool [F]) from the reference's cull_mesh on CPU."""
    from oracle import ref_harness
    ref_harness.install()
    import slam.common.common as rc
    V, nF = inp['verts'].shape[0], inp['faces'].shape[0]
    faces = np.concatenate([inp['faces'], np.repeat(np.arange(V)[:, None], 3, 1)])
    mesh = _RecordingMesh(inp['verts'], faces)
    est = [torch.from_numpy(p) for p in inp['est']] if use_est else None
    rc.cull_mesh(Dataset(inp['depth'], inp['poses'], inp['camera']), mesh, estimate_c2w_list=est,
                 eval_rec=eval_rec, truncation=truncation, device='cpu')
    return mesh.kept[nF:], mesh.kept[:nF]


def main():
    inp = inputs()
    out = dict(inp)
    for name, use_est, eval_rec, trunc in CASES:
        seen, kept = reference_decisions(inp, use_est, eval_rec, trunc)
        out[name + '_seen'], out[name + '_kept'] = seen, kept
        print(name, 'seen', int(seen.sum()), 'of', seen.size, 'kept faces', int(kept.sum()))
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'cull_mesh_ref.npz')
    np.savez_compressed(path, **out)
    print(path)


if __name__ == '__main__':
    main()
