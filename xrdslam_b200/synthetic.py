"""Synthetic 640x480 RGB-D sequence (SURVEY.md section 8d): an analytic room box
with two inner boxes, depth by exact ray/plane intersection, smooth procedural
colour, camera on a circle looking at the room centre (OpenGL c2w convention,
as the reference's loaders produce, slam/common/datasets.py:154-163)."""
from __future__ import annotations

import numpy as np

from .camera import Camera

ROOM = np.array([[-2.9, 2.9], [-3.9, 2.4], [-1.9, 2.4]])
BOXES = [np.array([[0.8, 1.8], [-0.2, 0.9], [-1.9, -0.7]]),
         np.array([[-2.0, -1.1], [-2.5, -1.3], [-1.9, 0.1]])]
CENTRE = np.array([0.0, -0.75, 0.25])


def make_camera(width=640, height=480):
    f = 320.0 * width / 640.0
    return Camera(f, f, (width - 1) / 2.0, (height - 1) / 2.0, width, height)


def look_at(eye, target, up=np.array([0.0, 0.0, 1.0])):
    f = target - eye
    f = f / np.linalg.norm(f)
    x = np.cross(f, up)
    x = x / np.linalg.norm(x)
    y = np.cross(x, f)
    c2w = np.eye(4)
    c2w[:3, 0], c2w[:3, 1], c2w[:3, 2], c2w[:3, 3] = x, y, -f, eye
    return c2w.astype(np.float32)


def trajectory(n_frames, radius=0.8, offset=(0.0, 0.0, 0.0), turn=0.25):
    """c2w of n_frames cameras on a circle: `turn` of a full revolution over the run."""
    poses = []
    for k in range(n_frames):
        a = 2 * np.pi * k / max(n_frames, 1) * turn
        eye = CENTRE + np.array([radius * np.cos(a), radius * np.sin(a), 0.1])
        tgt = CENTRE + np.array([-1.5 * np.cos(a + 0.6), -1.5 * np.sin(a + 0.6), -0.3])
        c2w = look_at(eye, tgt)
        c2w[:3, 3] += np.asarray(offset, dtype=np.float32)
        poses.append(c2w)
    return poses


def _slab(o, d, box):
    with np.errstate(divide='ignore', invalid='ignore'):
        t0 = (box[:, 0] - o) / d
        t1 = (box[:, 1] - o) / d
    tn = np.minimum(t0, t1).max(-1)
    tf = np.maximum(t0, t1).min(-1)
    return tn, tf


def render_frame(camera: Camera, c2w, offset=(0.0, 0.0, 0.0), invalid_frac=0.02,
                 seed=0):
    """-> rgb [H,W,3] f32 in [0,1], depth [H,W] f32 (z-depth, 0 = invalid)."""
    H, W = camera.height, camera.width
    j, i = np.meshgrid(np.arange(H, dtype=np.float64),
                       np.arange(W, dtype=np.float64), indexing='ij')
    dirs = np.stack([(i - camera.cx) / camera.fx, -(j - camera.cy) / camera.fy,
                     -np.ones_like(i)], -1)
    c2w = np.asarray(c2w, dtype=np.float64)
    off = np.asarray(offset, dtype=np.float64)
    d = dirs @ c2w[:3, :3].T
    o = c2w[:3, 3] - off
    _, t = _slab(o, d, ROOM)  # camera is inside: exit distance
    for b in BOXES:
        tn, tf = _slab(o, d, b)
        hit = (tn < tf) & (tn > 0)
        t = np.where(hit & (tn < t), tn, t)
    p = o + d * t[..., None]
    rgb = 0.5 + 0.5 * np.sin(p @ np.array([[2.1, 0.7, 1.3], [0.9, 2.3, 0.5],
                                           [1.1, 0.6, 2.7]]) + np.array([0.3, 1.1, 2.0]))
    depth = t.copy()  # |dir_z| == 1 -> ray parameter == z-depth
    rng = np.random.default_rng(seed)
    depth[rng.random((H, W)) < invalid_frac] = 0.0
    return rgb.astype(np.float32), depth.astype(np.float32)


def make_sequence(n_frames, width=640, height=480, offset=(0.0, 0.0, 0.0), turn=0.25):
    cam = make_camera(width, height)
    poses = trajectory(n_frames, offset=offset, turn=turn)
    frames = [render_frame(cam, p, offset=offset, seed=k)
              for k, p in enumerate(poses)]
    return cam, poses, frames


REPLICA_DEPTH_SCALE = 6553.5


def write_replica(folder, n_frames, width=640, height=480, offset=(0.0, 0.0, 0.0), turn=0.25):
    """The sequence of make_sequence as a Replica folder: results/frame%06d.jpg (colour, JPEG
    quality 95), results/depth%06d.png (uint16 depth x 6553.5), traj.txt (one row-major c2w per
    line in the dataset's camera axes: columns 1 and 2 negated, the inverse of the reader's flip)
    and devices.yaml.  -> (camera, poses)."""
    import os
    cam, poses, frames = make_sequence(n_frames, width=width, height=height, offset=offset,
                                       turn=turn)
    res = os.path.join(folder, 'results')
    os.makedirs(res, exist_ok=True)
    try:
        import cv2
    except ImportError:
        cv2 = None
    for k, (rgb, depth) in enumerate(frames):
        rgb8 = np.clip(np.rint(rgb * 255.0), 0, 255).astype(np.uint8)
        d16 = np.clip(np.rint(depth.astype(np.float64) * REPLICA_DEPTH_SCALE), 0,
                      65535).astype(np.uint16)
        cpath = os.path.join(res, f'frame{k:06d}.jpg')
        dpath = os.path.join(res, f'depth{k:06d}.png')
        if cv2 is not None:
            cv2.imwrite(cpath, rgb8[..., ::-1], [cv2.IMWRITE_JPEG_QUALITY, 95])
            cv2.imwrite(dpath, d16)
        else:
            from PIL import Image
            Image.fromarray(rgb8).save(cpath, quality=95)
            Image.fromarray(d16).save(dpath)
    with open(os.path.join(folder, 'traj.txt'), 'w') as f:
        for p in poses:
            q = np.asarray(p, np.float64).copy()
            q[:3, 1] *= -1
            q[:3, 2] *= -1
            f.write(' '.join(repr(float(v)) for v in q.reshape(-1)) + '\n')
    with open(os.path.join(folder, 'devices.yaml'), 'w') as f:
        f.write(f'cam:\n  H: {height}\n  W: {width}\n  fx: {cam.fx!r}\n  fy: {cam.fy!r}\n'
                f'  cx: {cam.cx!r}\n  cy: {cam.cy!r}\n  png_depth_scale: {REPLICA_DEPTH_SCALE}\n')
    return cam, poses


def _imwrite(path, img, quality=95):
    """uint8 BGR [H,W,3] (JPEG quality `quality` for .jpg) or uint16 [H,W] PNG."""
    try:
        import cv2
    except ImportError:
        cv2 = None
    if cv2 is not None:
        params = [cv2.IMWRITE_JPEG_QUALITY, quality] if path.endswith('.jpg') else []
        if not cv2.imwrite(path, img, params):
            raise OSError(f'could not write {path}')
        return
    from PIL import Image
    Image.fromarray(img[..., ::-1] if img.ndim == 3 else img).save(path, quality=quality)


def _layout_frames(n_frames, width, height, offset, turn, color_scale=1.0):
    """make_sequence's frames for a folder writer: -> (depth camera, poses, [(uint8 BGR colour,
    float32 depth in metres)]).  With color_scale != 1 the colour is rendered at
    (round(height s), round(width s)) through a camera with the same field of view, so resizing
    it to the depth's size (as the ingest does) lines it up with the depth."""
    cam, poses, frames = make_sequence(n_frames, width=width, height=height, offset=offset,
                                       turn=turn)
    Wc, Hc = int(round(width * color_scale)), int(round(height * color_scale))
    ccam = Camera(cam.fx * Wc / width, cam.fy * Hc / height, (Wc - 1) / 2.0, (Hc - 1) / 2.0,
                  Wc, Hc)
    out = []
    for k, (rgb, depth) in enumerate(frames):
        if (Hc, Wc) != (height, width):
            rgb, _ = render_frame(ccam, poses[k], offset=offset, seed=k)
        rgb8 = np.clip(np.rint(rgb * 255.0), 0, 255).astype(np.uint8)
        out.append((np.ascontiguousarray(rgb8[..., ::-1]), depth))
    return cam, poses, out


def _depth_u16(depth, scale):
    return np.clip(np.rint(depth.astype(np.float64) * scale), 0, 65535).astype(np.uint16)


def _dataset_axes(c2w):
    """c2w in the codebase's camera axes -> the dataset's (columns 1 and 2 negated), float64."""
    q = np.asarray(c2w, np.float64).copy()
    q[:3, 1] *= -1
    q[:3, 2] *= -1
    return q


def _write_devices(folder, cam, png_depth_scale, distortion=None, crop_edge=0,
                   downsample_factor=1):
    """devices.yaml: the depth camera, the depth scale and the optional ingest settings."""
    import os
    lines = ['cam:', f'  H: {cam.height}', f'  W: {cam.width}', f'  fx: {cam.fx!r}',
             f'  fy: {cam.fy!r}', f'  cx: {cam.cx!r}', f'  cy: {cam.cy!r}',
             f'  png_depth_scale: {png_depth_scale!r}']
    if distortion is not None:
        lines.append(f'  distortion: {[float(v) for v in distortion]!r}')
    if crop_edge:
        lines.append(f'  crop_edge: {int(crop_edge)}')
    if downsample_factor != 1:
        lines.append(f'  downsample_factor: {int(downsample_factor)}')
    with open(os.path.join(folder, 'devices.yaml'), 'w') as f:
        f.write('\n'.join(lines) + '\n')


TUM_DEPTH_SCALE = 5000.0
METRIC_MM_DEPTH_SCALE = 1000.0  # ScanNet, 7-Scenes and Azure Kinect store millimetres


def write_tum(folder, n_frames, width=640, height=480, offset=(0.0, 0.0, 0.0), turn=0.25,
              distortion=None, crop_edge=0, downsample_factor=1, seed=0):
    """The sequence as a TUM RGB-D folder: rgb/<t>.png, depth/<t>.png (uint16 depth x 5000),
    rgb.txt, depth.txt and groundtruth.txt (tx ty tz qx qy qz qw) with TUM's '#' headers, and
    devices.yaml.  Frame k is taken at about 0.1 k s (after frame 1, 0.5 s later), with jittered
    image, depth and pose timestamps.  Three extra images exercise the reader's association:
    one 0.02 s after frame 0 (with its own depth and closer than 1/32 s, so the frame-rate
    subsampling drops it), one in the gap after frame 1 with no depth within 0.08 s, and one there
    with a depth image but no pose within 0.08 s.  The reader keeps exactly the n_frames frames.
    -> (camera, poses)."""
    import os
    from scipy.spatial.transform import Rotation
    if n_frames < 2:
        raise ValueError('write_tum needs at least 2 frames')
    cam, poses, frames = _layout_frames(n_frames, width, height, offset, turn)
    rng = np.random.default_rng(seed)
    t0 = 1305031102.0
    t_img = t0 + 0.1 * np.arange(n_frames) + rng.uniform(-0.01, 0.01, n_frames)
    t_img[2:] += 0.5
    t_dep = t_img + rng.uniform(-0.004, 0.004, n_frames)
    t_pose = t_img + rng.uniform(-0.01, 0.01, n_frames)
    os.makedirs(os.path.join(folder, 'rgb'), exist_ok=True)
    os.makedirs(os.path.join(folder, 'depth'), exist_ok=True)
    rgb_rows, depth_rows = [], []

    def add(t_rgb, color, t_depth=None, depth=None):
        name = f'rgb/{t_rgb:.6f}.png'
        _imwrite(os.path.join(folder, name), color)
        rgb_rows.append((t_rgb, name))
        if depth is not None:
            dname = f'depth/{t_depth:.6f}.png'
            _imwrite(os.path.join(folder, dname), _depth_u16(depth, TUM_DEPTH_SCALE))
            depth_rows.append((t_depth, dname))

    for k, (color, depth) in enumerate(frames):
        add(t_img[k], color, t_dep[k], depth)
    gap = t_img[1]
    add(t_img[0] + 0.02, frames[0][0], t_img[0] + 0.02, frames[0][1])  # too soon after frame 0
    add(gap + 0.25, frames[1][0])                                      # no depth
    add(gap + 0.4, frames[1][0], gap + 0.4, frames[1][1])              # no pose
    for name, rows in (('rgb', rgb_rows), ('depth', depth_rows)):
        with open(os.path.join(folder, f'{name}.txt'), 'w') as f:
            f.write(f'# {name} maps\n# file: synthetic\n# timestamp filename\n')
            for t, path in sorted(rows):
                f.write(f'{t:.6f} {path}\n')
    with open(os.path.join(folder, 'groundtruth.txt'), 'w') as f:
        f.write('# ground truth trajectory\n# file: synthetic\n# timestamp tx ty tz qx qy qz qw\n')
        for t, p in zip(t_pose, poses):
            q = _dataset_axes(p)
            vals = list(q[:3, 3]) + list(Rotation.from_matrix(q[:3, :3]).as_quat())
            f.write(f'{t:.4f} ' + ' '.join(f'{v:.17g}' for v in vals) + '\n')
    _write_devices(folder, cam, TUM_DEPTH_SCALE, distortion, crop_edge, downsample_factor)
    return cam, poses


def write_scannet(folder, n_frames, width=640, height=480, offset=(0.0, 0.0, 0.0), turn=0.25,
                  color_scale=2.0, distortion=None, crop_edge=0, downsample_factor=1):
    """The sequence as a ScanNet folder: devices.yaml, frames/color/<k>.jpg (colour_scale times
    the depth's size), frames/depth/<k>.png (uint16 millimetres), frames/pose/<k>.txt (four
    space-separated rows), with unpadded frame numbers.  -> (camera, poses)."""
    import os
    cam, poses, frames = _layout_frames(n_frames, width, height, offset, turn, color_scale)
    base = os.path.join(folder, 'frames')
    for sub in ('color', 'depth', 'pose'):
        os.makedirs(os.path.join(base, sub), exist_ok=True)
    for k, ((color, depth), p) in enumerate(zip(frames, poses)):
        _imwrite(os.path.join(base, 'color', f'{k}.jpg'), color)
        _imwrite(os.path.join(base, 'depth', f'{k}.png'), _depth_u16(depth, METRIC_MM_DEPTH_SCALE))
        with open(os.path.join(base, 'pose', f'{k}.txt'), 'w') as f:
            for row in _dataset_axes(p):
                f.write(' '.join(repr(float(v)) for v in row) + '\n')
    _write_devices(folder, cam, METRIC_MM_DEPTH_SCALE, distortion, crop_edge, downsample_factor)
    return cam, poses


def write_7scenes(folder, n_frames, width=640, height=480, offset=(0.0, 0.0, 0.0), turn=0.25,
                  distortion=None, crop_edge=0, downsample_factor=1):
    """The sequence as a 7-Scenes sequence folder: frame-%06d.color.png, frame-%06d.depth.png
    (uint16 millimetres) and frame-%06d.pose.txt (four tab-separated rows), and devices.yaml.
    -> (camera, poses)."""
    import os
    cam, poses, frames = _layout_frames(n_frames, width, height, offset, turn)
    os.makedirs(folder, exist_ok=True)
    for k, ((color, depth), p) in enumerate(zip(frames, poses)):
        stem = os.path.join(folder, f'frame-{k:06d}')
        _imwrite(stem + '.color.png', color)
        _imwrite(stem + '.depth.png', _depth_u16(depth, METRIC_MM_DEPTH_SCALE))
        with open(stem + '.pose.txt', 'w') as f:
            for row in _dataset_axes(p):
                f.write('\t'.join(f'{float(v):.17g}' for v in row) + '\t\n')
    _write_devices(folder, cam, METRIC_MM_DEPTH_SCALE, distortion, crop_edge, downsample_factor)
    return cam, poses


def write_azure(folder, n_frames, width=640, height=480, offset=(0.0, 0.0, 0.0), turn=0.25,
                color_scale=1.5, trajectory_log=True, distortion=None, crop_edge=0,
                downsample_factor=1):
    """The sequence as an Azure Kinect folder: color/%05d.jpg (color_scale times the depth's
    size), depth/%05d.png (uint16 millimetres), scene/trajectory.log (5-line blocks: 'k k n',
    then the four rows; left out with trajectory_log=False) and devices.yaml.
    -> (camera, poses)."""
    import os
    cam, poses, frames = _layout_frames(n_frames, width, height, offset, turn, color_scale)
    for sub in ('color', 'depth', 'scene'):
        os.makedirs(os.path.join(folder, sub), exist_ok=True)
    for k, (color, depth) in enumerate(frames):
        _imwrite(os.path.join(folder, 'color', f'{k:05d}.jpg'), color)
        _imwrite(os.path.join(folder, 'depth', f'{k:05d}.png'),
                 _depth_u16(depth, METRIC_MM_DEPTH_SCALE))
    if trajectory_log:
        with open(os.path.join(folder, 'scene', 'trajectory.log'), 'w') as f:
            for k, p in enumerate(poses):
                f.write(f'{k} {k} {n_frames}\n')
                for row in _dataset_axes(p):
                    f.write(' '.join(f'{float(v):.17g}' for v in row) + '\n')
    _write_devices(folder, cam, METRIC_MM_DEPTH_SCALE, distortion, crop_edge, downsample_factor)
    return cam, poses


def write_cofusion(folder, n_frames, width=640, height=480, offset=(0.0, 0.0, 0.0), turn=0.25,
                   nan_frac=0.01, distortion=None, crop_edge=0, downsample_factor=1, seed=0):
    """The sequence as a CoFusion folder: colour/Color%04d.png and depth_noise/Depth%04d.exr
    (float32 metres in the 'Y' channel, png_depth_scale 1; about nan_frac of the pixels NaN on
    top of make_sequence's invalid zeros), and devices.yaml.  CoFusion's reader gives identity
    poses, so the trajectory is not written.  Needs cv2's OpenEXR codec.  -> (camera, poses)."""
    import os
    os.environ.setdefault('OPENCV_IO_ENABLE_OPENEXR', '1')
    import cv2
    cam, poses, frames = _layout_frames(n_frames, width, height, offset, turn)
    for sub in ('colour', 'depth_noise'):
        os.makedirs(os.path.join(folder, sub), exist_ok=True)
    rng = np.random.default_rng(seed)
    for k, (color, depth) in enumerate(frames):
        _imwrite(os.path.join(folder, 'colour', f'Color{k:04d}.png'), color)
        d = depth.astype(np.float32).copy()
        d[rng.random(d.shape) < nan_frac] = np.nan
        path = os.path.join(folder, 'depth_noise', f'Depth{k:04d}.exr')
        if not cv2.imwrite(path, d):
            raise OSError(f'could not write {path}')
    _write_devices(folder, cam, 1.0, distortion, crop_edge, downsample_factor)
    return cam, poses


def _grid_rect(origin, u, v, nu, nv):
    """A rectangle origin + [0,1]u + [0,1]v as an (nu x nv)-cell triangle grid."""
    a, b = np.meshgrid(np.linspace(0.0, 1.0, nu + 1), np.linspace(0.0, 1.0, nv + 1), indexing='ij')
    verts = origin + a.reshape(-1, 1) * u + b.reshape(-1, 1) * v
    idx = np.arange((nu + 1) * (nv + 1)).reshape(nu + 1, nv + 1)
    q = np.stack([idx[:-1, :-1], idx[1:, :-1], idx[1:, 1:], idx[:-1, 1:]], -1).reshape(-1, 4)
    faces = np.concatenate([q[:, [0, 1, 2]], q[:, [0, 2, 3]]])
    return verts, faces


def room_mesh(spacing=0.1):
    """The analytic scene (ROOM's six walls and the BOXES' faces that do not lie on a wall) as a
    triangle mesh with vertices about `spacing` apart: -> (verts f32 [V,3], faces i32 [F,3]).
    The ground truth the reconstruction tests score against."""
    verts, faces, base = [], [], 0

    def box_faces(box, skip_walls):
        for ax in range(3):
            u_ax, v_ax = [a for a in range(3) if a != ax]
            for side in range(2):
                if skip_walls and box[ax, side] in (ROOM[ax, 0], ROOM[ax, 1]):
                    continue
                o = box[:, 0].astype(np.float64).copy()
                o[ax] = box[ax, side]
                u = np.zeros(3)
                v = np.zeros(3)
                u[u_ax] = box[u_ax, 1] - box[u_ax, 0]
                v[v_ax] = box[v_ax, 1] - box[v_ax, 0]
                yield o, u, v

    rects = list(box_faces(ROOM, False))
    for b in BOXES:
        rects += list(box_faces(b, True))
    for o, u, v in rects:
        nu = max(1, int(round(np.linalg.norm(u) / spacing)))
        nv = max(1, int(round(np.linalg.norm(v) / spacing)))
        vv, ff = _grid_rect(o, u, v, nu, nv)
        verts.append(vv)
        faces.append(ff + base)
        base += len(vv)
    return np.concatenate(verts).astype(np.float32), np.concatenate(faces).astype(np.int32)
