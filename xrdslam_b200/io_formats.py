"""On-disk artefacts the reference's tracker writes for `ds-eval` (SURVEY row f4;
slam/pipeline/tracker.py:258-278, 388-420; scripts/eval.py:36-50): the trajectory checkpoint
`eval.tar` and binary PLY files for meshes (`final_mesh.ply`, what `trimesh.Trimesh.export`
produces) and point clouds (`cloud/%05d.ply`, what `o3d.io.write_point_cloud` produces).
Host-side I/O only; trimesh / open3d are not needed to write or read these."""
from __future__ import annotations

import os

import numpy as np
import torch


def save_eval_tar(algorithm, out_dir, idx):
    """tracker.py:269-278 / 410-420: {'gt_c2w_list_ori', 'gt_c2w_list', 'estimate_c2w_list',
    'idx'} in torch's legacy (non-zipfile) serialization -> `<out_dir>/eval.tar`."""
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, 'eval.tar')
    cpu = lambda lst: [t.detach().cpu() if torch.is_tensor(t) else torch.as_tensor(np.asarray(t))
                       for t in lst]
    torch.save({'gt_c2w_list_ori': cpu(algorithm.get_gt_c2w_list_ori()),
                'gt_c2w_list': cpu(algorithm.get_gt_c2w_list()),
                'estimate_c2w_list': cpu(algorithm.get_estimate_c2w_list()),
                'idx': idx if torch.is_tensor(idx) else torch.tensor(int(idx))},
               path, _use_new_zipfile_serialization=False)
    return path


def load_eval_tar(path):
    """scripts/eval.py:42-46: -> (estimate_c2w_list, gt_c2w_list_ori, N)."""
    ckpt = torch.load(path, map_location=torch.device('cpu'), weights_only=False)
    return ckpt['estimate_c2w_list'], ckpt['gt_c2w_list_ori'], int(ckpt['idx'])


def valid_pose_mask(c2w_list, n):
    """scripts/utils/eval_ate.py:321-339: ground-truth poses holding inf / nan are masked out."""
    m = torch.ones(n, dtype=torch.bool)
    for i in range(n):
        t = torch.as_tensor(c2w_list[i])
        if torch.isinf(t).any() or torch.isnan(t).any():
            m[i] = False
    return m


def ate_rmse(gt_c2w_list, est_c2w_list, n=None, correct_scale=False):
    """Absolute trajectory error after the closed-form rigid (Horn / Umeyama) alignment of the
    estimated camera centres onto the ground truth (scripts/utils/eval_ate.py `align` +
    `evaluate`): -> dict(rmse, mean, median, max, rot [3,3], trans [3], scale)."""
    n = len(gt_c2w_list) if n is None else n
    m = valid_pose_mask(gt_c2w_list, n)
    gt = np.stack([np.asarray(torch.as_tensor(gt_c2w_list[i]))[:3, 3] for i in range(n) if m[i]]).T
    est = np.stack([np.asarray(torch.as_tensor(est_c2w_list[i]))[:3, 3] for i in range(n) if m[i]]).T
    gt, est = gt.astype(np.float64), est.astype(np.float64)
    mu_g, mu_e = gt.mean(1, keepdims=True), est.mean(1, keepdims=True)
    g0, e0 = gt - mu_g, est - mu_e
    W = e0 @ g0.T  # sum of outer(model, data)
    U, d, Vt = np.linalg.svd(W.T)
    S = np.eye(3)
    if np.linalg.det(U) * np.linalg.det(Vt) < 0:
        S[2, 2] = -1
    rot = U @ S @ Vt
    scale = 1.0
    if correct_scale:
        re = rot @ e0
        scale = float((g0 * re).sum() / (re * re).sum())
    trans = mu_g - scale * rot @ mu_e
    err = np.sqrt((((scale * rot @ est + trans) - gt) ** 2).sum(0))
    return dict(rmse=float(np.sqrt((err ** 2).mean())), mean=float(err.mean()),
                median=float(np.median(err)), max=float(err.max()), rot=rot, trans=trans.reshape(3),
                scale=scale)


def write_ply(path, vertices, faces=None, colors=None):
    """Binary little-endian PLY: float32 x y z [+ uchar red green blue (alpha 255 for meshes)]
    per vertex and, for meshes, `list uchar int vertex_indices` faces -- the layouts trimesh and
    open3d write.  colors: float in [0,1] or uint8."""
    v = np.ascontiguousarray(np.asarray(vertices, dtype=np.float32).reshape(-1, 3))
    c = None
    if colors is not None:
        c = np.asarray(colors)
        if c.dtype != np.uint8:
            c = np.clip(np.round(c.astype(np.float64) * 255.0), 0, 255).astype(np.uint8)
        c = c.reshape(-1, c.shape[-1])[:, :3]
        assert c.shape[0] == v.shape[0]
    f = None if faces is None else np.ascontiguousarray(np.asarray(faces, dtype=np.int32).reshape(-1, 3))
    mesh = f is not None
    hdr = ['ply', 'format binary_little_endian 1.0', f'element vertex {v.shape[0]}',
           'property float x', 'property float y', 'property float z']
    if c is not None:
        hdr += ['property uchar red', 'property uchar green', 'property uchar blue']
        if mesh:
            hdr += ['property uchar alpha']
    if mesh:
        hdr += [f'element face {f.shape[0]}', 'property list uchar int vertex_indices']
    hdr += ['end_header']
    fields = [('x', '<f4'), ('y', '<f4'), ('z', '<f4')]
    if c is not None:
        fields += [('r', 'u1'), ('g', 'u1'), ('b', 'u1')] + ([('a', 'u1')] if mesh else [])
    rec = np.empty(v.shape[0], dtype=np.dtype(fields))
    rec['x'], rec['y'], rec['z'] = v[:, 0], v[:, 1], v[:, 2]
    if c is not None:
        rec['r'], rec['g'], rec['b'] = c[:, 0], c[:, 1], c[:, 2]
        if mesh:
            rec['a'] = 255
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    with open(path, 'wb') as fh:
        fh.write(('\n'.join(hdr) + '\n').encode('ascii'))
        fh.write(rec.tobytes())
        if mesh:
            fr = np.empty(f.shape[0], dtype=np.dtype([('n', 'u1'), ('i', '<i4', (3,))]))
            fr['n'] = 3
            fr['i'] = f
            fh.write(fr.tobytes())
    return path


_PLY_SCALARS = {'char': 'i1', 'int8': 'i1', 'uchar': 'u1', 'uint8': 'u1', 'short': '<i2',
                'int16': '<i2', 'ushort': '<u2', 'uint16': '<u2', 'int': '<i4', 'int32': '<i4',
                'uint': '<u4', 'uint32': '<u4', 'float': '<f4', 'float32': '<f4',
                'double': '<f8', 'float64': '<f8'}
_PLY_COUNTS = ('uchar', 'uint8', 'ushort', 'uint16', 'int', 'int32', 'uint', 'uint32')
_PLY_INDICES = ('int', 'int32', 'uint', 'uint32')


def read_ply(path):
    """Binary little-endian PLY reader: the files `write_ply` (and trimesh / open3d with the same
    properties) produce and ground-truth meshes as Replica ships them.  Vertex properties may be
    any scalar type; faces are `list uchar|ushort|int|uint int|uint vertex_indices|vertex_index`
    with any other face properties (scalars or lists) skipped.  ASCII and big-endian files and
    other elements after the faces' are rejected with ValueError.
    -> (vertices f32 [n,3], faces i32 [m,3] or None, colors u8 [n,3] or None)."""
    with open(path, 'rb') as fh:
        data = fh.read()
    if not data.startswith(b'ply'):
        raise ValueError(f'{path}: not a PLY file')
    try:
        end = data.index(b'end_header\n') + len(b'end_header\n')
    except ValueError:
        raise ValueError(f'{path}: PLY header has no end_header') from None
    lines = [ln.strip() for ln in data[:end].decode('ascii').strip().split('\n')]
    fmt = lines[1].split()
    if fmt[:2] != ['format', 'binary_little_endian']:
        raise ValueError(f'{path}: only binary_little_endian PLY is read, not {lines[1]!r}')
    elements, cur = [], None
    for ln in lines[2:]:
        t = ln.split()
        if not t or t[0] in ('comment', 'obj_info', 'end_header'):
            continue
        if t[0] == 'element':
            cur = (t[1], int(t[2]), [])
            elements.append(cur)
        elif t[0] == 'property':
            if cur is None:
                raise ValueError(f'{path}: property before any element')
            if t[1] == 'list':
                if t[2] not in _PLY_SCALARS or t[3] not in _PLY_SCALARS:
                    raise ValueError(f'{path}: unsupported list property {ln!r}')
                cur[2].append(('list', t[4], t[2], t[3]))
            else:
                if t[1] not in _PLY_SCALARS:
                    raise ValueError(f'{path}: unsupported property type {ln!r}')
                cur[2].append(('scalar', t[2], t[1]))
    off = end
    v = f = c = None
    for name, count, props in elements:
        if name == 'vertex':
            if any(p[0] == 'list' for p in props):
                raise ValueError(f'{path}: list properties on vertices are not supported')
            dt = np.dtype([(p[1], _PLY_SCALARS[p[2]]) for p in props])
            rec = np.frombuffer(data, dtype=dt, count=count, offset=off)
            off += count * dt.itemsize
            v = np.stack([rec['x'], rec['y'], rec['z']], -1).astype(np.float32)
            if 'red' in dt.names:
                c = np.stack([rec['red'], rec['green'], rec['blue']], -1).astype(np.uint8)
        elif name == 'face':
            f, off = _read_faces(path, data, off, count, props)
        elif count:
            raise ValueError(f'{path}: unsupported element {name!r}')
    if v is None:
        raise ValueError(f'{path}: no vertex element')
    return v, (f if f is not None and len(f) else None), c


def _read_faces(path, data, off, count, props):
    lists = [p for p in props if p[0] == 'list' and p[1] in ('vertex_indices', 'vertex_index')]
    if len(lists) != 1 or lists[0][2] not in _PLY_COUNTS or lists[0][3] not in _PLY_INDICES:
        raise ValueError(f'{path}: faces need one list uchar|ushort|int|uint int|uint '
                         'vertex_indices property')
    if all(p[0] == 'scalar' or p is lists[0] for p in props):
        # fixed-size records when every face is a triangle: one vectorised read
        fields = []
        for k, p in enumerate(props):
            if p is lists[0]:
                fields += [('n', _PLY_SCALARS[p[2]]), ('i', _PLY_SCALARS[p[3]], (3,))]
            else:
                fields.append((f's{k}', _PLY_SCALARS[p[2]]))
        fdt = np.dtype(fields)
        if off + count * fdt.itemsize <= len(data):
            rec = np.frombuffer(data, dtype=fdt, count=count, offset=off)
            if count == 0 or np.all(rec['n'] == 3):
                return rec['i'].astype(np.int32), off + count * fdt.itemsize
    faces = np.empty((count, 3), np.int32)
    for r in range(count):
        for p in props:
            if p[0] == 'scalar':
                off += np.dtype(_PLY_SCALARS[p[2]]).itemsize
                continue
            cdt, idt = np.dtype(_PLY_SCALARS[p[2]]), np.dtype(_PLY_SCALARS[p[3]])
            n = int(np.frombuffer(data, cdt, 1, off)[0])
            off += cdt.itemsize
            vals = np.frombuffer(data, idt, n, off)
            off += n * idt.itemsize
            if p is lists[0]:
                if n != 3:
                    raise ValueError(f'{path}: face {r} has {n} vertices, only triangles are read')
                faces[r] = vals
    return faces, off
