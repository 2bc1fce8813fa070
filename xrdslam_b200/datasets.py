"""RGB-D dataset readers (slam/common/datasets.py): the Replica, TUM RGB-D, ScanNet, 7-Scenes,
Azure Kinect and CoFusion folder layouts, decoded on the host and turned into float32 device
frames by one CUDA call (csrc/ingest.cu, `frame_ingest`).

`dataset[i]` returns `(i, rgb f32 [h,w,3], depth f32 [h,w], c2w f32 [4,4])` as device tensors,
the protocol of the reference's BaseDataset.__getitem__ (datasets.py:95-134).  The colour is
undistorted, converted, resized, cropped and downsampled exactly as that method does with cv2
(see include/xrdslam_b200.h, xrd_frame_ingest).

Decoding uses cv2.imread when cv2 is importable, as the reference does; otherwise PIL, whose
JPEG decoder may round differently from cv2's libjpeg build, so the pixels then match the
reference's only up to the decoder.  `DECODER` names the one in use.

Iterating a dataset in order prefetches: a host thread decodes frame i + 1 into pinned memory
while frame i is being used (the reference's DataLoader(num_workers=1), without its float64 host
work).

The readers differ only in file listing, sort order and pose parsing, which follow the reference's
classes line by line (`dataset_dict`): poses are built in float64 and handed out as float32
tensors.  Depth is a 16-bit PNG (`xrd_frame_ingest`) or, for CoFusion, the float32 'Y' channel of
an OpenEXR file read through cv2 (`xrd_frame_ingest_f32`).  Colour that the ingest resizes with
INTER_LINEAR (ScanNet's and Azure's frames are larger than their depth) equals cv2 built without
Intel IPP bit for bit; a cv2 built with IPP differs by up to about 2e-6 there.  EuRoC
(monocular + IMU, read only by DPVO) is not supported."""
from __future__ import annotations

import glob
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from .camera import Camera

try:
    import cv2
    DECODER = 'cv2'
except ImportError:  # pragma: no cover - depends on the environment
    cv2 = None
    DECODER = 'PIL'


def read_color(path):
    """uint8 [H,W,3] in BGR order, as cv2.imread(path) returns it."""
    if cv2 is not None:
        img = cv2.imread(path)
        if img is None:
            raise FileNotFoundError(path)
        return img
    from PIL import Image
    with Image.open(path) as im:
        return np.ascontiguousarray(np.asarray(im.convert('RGB'))[..., ::-1])


def read_depth(path):
    """uint16 [H,W], as cv2.imread(path, cv2.IMREAD_UNCHANGED) returns a 16-bit PNG."""
    if cv2 is not None:
        img = cv2.imread(path, cv2.IMREAD_UNCHANGED)
        if img is None:
            raise FileNotFoundError(path)
    else:
        from PIL import Image
        with Image.open(path) as im:
            img = np.asarray(im)
    if img.dtype != np.uint16 or img.ndim != 2:
        raise ValueError(f'{path}: expected a 16-bit single-channel PNG, got {img.dtype} '
                         f'{img.shape}')
    return img


def read_depth_exr(path):
    """float32 [H,W]: the 'Y' channel of a single-channel OpenEXR file (datasets.py:20-52,
    readEXR_onlydepth), decoded by cv2 with its OpenEXR codec enabled.  Every bit of the stored
    values is kept, NaN payloads included.  Raises where the reference's reader returns None."""
    if cv2 is None:
        raise RuntimeError(f'{path}: reading OpenEXR depth needs cv2')
    # cv2 reads this switch once, at its first OpenEXR access; a user's own setting is kept
    os.environ.setdefault('OPENCV_IO_ENABLE_OPENEXR', '1')
    try:
        img = cv2.imread(path, cv2.IMREAD_UNCHANGED)
    except cv2.error as e:
        raise RuntimeError(f'{path}: cv2 cannot decode OpenEXR ({e}); it needs '
                           'OPENCV_IO_ENABLE_OPENEXR=1 before its first OpenEXR access') from e
    if img is None:
        if not os.path.exists(path):
            raise FileNotFoundError(path)
        raise RuntimeError(f'{path}: cv2 could not decode this OpenEXR file')
    if img.dtype != np.float32 or img.ndim != 2:
        raise ValueError(f'{path}: expected a single-channel (Y) float32 OpenEXR depth image, got '
                         f'{img.dtype} {img.shape}')
    return img


def read_depth_any(path):
    """The depth image of `path` as datasets.py:99-102 picks its decoder (by '.png' / '.exr' in
    the path): uint16 [H,W] or float32 [H,W]."""
    if '.png' in path:
        return read_depth(path)
    if '.exr' in path:
        return read_depth_exr(path)
    raise ValueError(f'{path}: depth must be a .png or an .exr file')


def ingest_config(B, color_shape, depth_shape, fx, fy, cx, cy, distortion=None,
                  png_depth_scale=6553.5, crop_edge=0, downsample_factor=1):
    from . import _cabi
    cfg = _cabi.XrdIngestCfg()
    cfg.B = B
    cfg.H0, cfg.W0 = int(color_shape[0]), int(color_shape[1])
    cfg.Hd, cfg.Wd = int(depth_shape[0]), int(depth_shape[1])
    cfg.fx, cfg.fy, cfg.cx, cfg.cy = float(fx), float(fy), float(cx), float(cy)
    dist = [] if distortion is None else [float(v) for v in np.asarray(distortion).ravel()]
    if len(dist) > 12:
        raise ValueError(f'{len(dist)} distortion coefficients (at most 12 are supported)')
    for k, v in enumerate(dist):
        cfg.dist[k] = v
    cfg.n_dist = len(dist)
    cfg.png_depth_scale = float(png_depth_scale)
    cfg.crop_edge, cfg.downsample_factor = int(crop_edge), int(downsample_factor)
    return cfg


def output_size(depth_shape, crop_edge=0, downsample_factor=1):
    """(h, w) of the frames made from depth images of `depth_shape`."""
    h, w = depth_shape[0] - 2 * crop_edge, depth_shape[1] - 2 * crop_edge
    if downsample_factor > 1:
        h, w = h // downsample_factor, w // downsample_factor
    return h, w


def frame_ingest(color, depth, fx, fy, cx, cy, distortion=None, png_depth_scale=6553.5,
                 crop_edge=0, downsample_factor=1, out=None):
    """B decoded frames on the device -> (rgb f32 [B,h,w,3], depth f32 [B,h,w]) on the device.

    color: uint8 [B,H0,W0,3] (BGR, cv2.imread's order); depth [B,Hd,Wd]: uint16 or int16 (same
    bits) from PNG, through xrd_frame_ingest, or float32 from OpenEXR, through
    xrd_frame_ingest_f32.  One or two launches on the current stream, no host synchronisation.
    `out` may hold preallocated (rgb, depth) tensors."""
    from . import _cabi
    if color.dim() == 3:
        color, depth = color[None], depth[None]
    if depth.dtype == torch.float32:
        entry = 'xrd_frame_ingest_f32'
    elif depth.dtype in (torch.int16, torch.uint16):
        entry = 'xrd_frame_ingest'
    else:
        raise TypeError(f'frame_ingest needs 16-bit or float32 depth, got {depth.dtype}')
    if color.dtype != torch.uint8:
        raise TypeError(f'frame_ingest needs uint8 colour, got {color.dtype}')
    if color.device.type != 'cuda' or depth.device != color.device:
        raise ValueError('frame_ingest needs both images on the same CUDA device')
    B = color.shape[0]
    if color.shape[-1] != 3 or depth.shape[0] != B:
        raise ValueError(f'shapes {tuple(color.shape)} / {tuple(depth.shape)}')
    cfg = ingest_config(B, color.shape[1:3], depth.shape[1:3], fx, fy, cx, cy, distortion,
                        png_depth_scale, crop_edge, downsample_factor)
    h, w = output_size(depth.shape[1:3], crop_edge, downsample_factor)
    if h < 1 or w < 1:
        raise ValueError(f'crop_edge {crop_edge} / downsample_factor {downsample_factor} leave '
                         f'no pixels of a {tuple(depth.shape[1:3])} depth image')
    color, depth = color.contiguous(), depth.contiguous()
    dev = color.device
    if out is None:
        rgb = torch.empty(B, h, w, 3, dtype=torch.float32, device=dev)
        dep = torch.empty(B, h, w, dtype=torch.float32, device=dev)
    else:
        rgb, dep = out
    ws, nbytes = _cabi.workspace(dev, 'frame_ingest', cfg)
    _cabi.launch_on(dev, entry, cfg, _cabi.ptr(color), _cabi.ptr(depth),
                    _cabi.ptr(rgb), _cabi.ptr(dep), _cabi.ptr(ws), nbytes)
    return rgb, dep


EUROC_UNSUPPORTED = ("the 'euroc' layout (datasets.py:170-173) is monocular images plus IMU "
                     "(data_format 'MonoImu'), read only by DPVO; none of this package's RGB-D "
                     'algorithms can consume it')


def get_dataset(data_path, data_type, device='cuda:0'):
    if data_type == 'euroc':
        raise NotImplementedError(EUROC_UNSUPPORTED)
    if data_type not in dataset_dict:
        raise ValueError(f'unknown data_type {data_type!r}; one of {sorted(dataset_dict)}')
    return dataset_dict[data_type](data_path, device=device)


def update_recursive(dict1, dict2):
    """slam/utils/config.py:41-52: merge dict2 into dict1, nested dicts key by key."""
    for k, v in dict2.items():
        if k not in dict1:
            dict1[k] = dict()
        if isinstance(v, dict):
            update_recursive(dict1[k], v)
        else:
            dict1[k] = v


def load_config(path):
    """slam/utils/config.py:6-38: a YAML file, merged recursively over the file its
    `inherit_from` names (NICE-SLAM's per-scene devices.yaml files inherit a dataset-wide one).
    A relative `inherit_from` is looked up from the working directory, as the reference does, and
    then next to the including file."""
    import yaml
    with open(path) as f:
        cfg_special = yaml.safe_load(f) or {}
    inherit_from = cfg_special.get('inherit_from')
    cfg = {}
    if inherit_from is not None:
        parent = str(inherit_from)
        if not os.path.isabs(parent) and not os.path.exists(parent):
            parent = os.path.join(os.path.dirname(os.path.abspath(path)), parent)
        cfg = load_config(parent)
    update_recursive(cfg, cfg_special)
    return cfg


class BaseDataset:
    """datasets.py:60-137: devices.yaml -> camera after crop / downsample (int() truncation as
    the reference); frames through `frame_ingest`."""

    def __init__(self, data_path, device='cuda:0'):
        self.data_format = 'RGBD'
        self.input_folder = str(data_path)
        self.device_yml = os.path.join(self.input_folder, 'devices.yaml')
        cfg = load_config(self.device_yml)
        self.cfg = cfg
        self.device = device
        cam = cfg['cam']
        self.png_depth_scale = cam['png_depth_scale']
        self.H, self.W, self.fx, self.fy, self.cx, self.cy = (cam['H'], cam['W'], cam['fx'],
                                                              cam['fy'], cam['cx'], cam['cy'])
        self.distortion = np.array(cam['distortion']) if 'distortion' in cam else None
        self.crop_edge = cam['crop_edge'] if 'crop_edge' in cam else 0
        self.downsample_factor = cam['downsample_factor'] if 'downsample_factor' in cam else 1
        f, e = self.downsample_factor, self.crop_edge
        self.camera = Camera(fx=self.fx / f, fy=self.fy / f, cx=(self.cx - e) / f,
                             cy=(self.cy - e) / f, height=int((self.H - 2 * e) / f),
                             width=int((self.W - 2 * e) / f))

    def __len__(self):
        return self.n_img

    def get_camera(self):
        return self.camera

    def read_raw(self, index):
        """Decoded frame `index` in pinned host memory: (uint8 BGR [H0,W0,3], int16 [Hd,Wd]
        holding the uint16 depth bits, or float32 [Hd,Wd] from an OpenEXR file)."""
        color = read_color(self.color_paths[index])
        depth = read_depth_any(self.depth_paths[index])
        if depth.dtype == np.uint16:
            depth = depth.view(np.int16)
        color, depth = torch.from_numpy(color), torch.from_numpy(depth)
        if torch.cuda.is_available():
            color, depth = color.pin_memory(), depth.pin_memory()
        return color, depth

    def ingest(self, index, raw):
        color, depth = raw
        dev = torch.device(self.device)
        rgb, dep = frame_ingest(color.to(dev, non_blocking=True),
                                depth.to(dev, non_blocking=True), self.fx, self.fy, self.cx,
                                self.cy, self.distortion, self.png_depth_scale, self.crop_edge,
                                self.downsample_factor)
        return index, rgb[0], dep[0], self.poses[index].to(dev)

    def __getitem__(self, index):
        if index < 0:
            index += len(self)
        if not 0 <= index < len(self):
            raise IndexError(index)
        return self.ingest(index, self.read_raw(index))

    def __iter__(self):
        """Frames in order; frame i + 1 is decoded on a host thread while frame i is used."""
        n = len(self)
        if n == 0:
            return
        with ThreadPoolExecutor(max_workers=1) as pool:
            nxt = pool.submit(self.read_raw, 0)
            for i in range(n):
                raw = nxt.result()
                if i + 1 < n:
                    nxt = pool.submit(self.read_raw, i + 1)
                yield self.ingest(i, raw)


def load_replica_poses(path, n_img):
    """datasets.py:150-167: row-major 4x4 c2w per line, columns 1 and 2 of the rotation negated
    (OpenCV -> the codebase's OpenGL camera axes), as float32 tensors."""
    poses = []
    with open(path) as f:
        lines = f.readlines()
    for i in range(n_img):
        c2w = np.array(list(map(float, lines[i].split()))).reshape(4, 4)
        c2w[:3, 1] *= -1
        c2w[:3, 2] *= -1
        poses.append(torch.from_numpy(c2w).float())
    return poses


class Replica(BaseDataset):
    def __init__(self, data_path, device='cuda:0'):
        super().__init__(data_path, device)
        self.color_paths = sorted(glob.glob(f'{self.input_folder}/results/frame*.jpg'))
        self.depth_paths = sorted(glob.glob(f'{self.input_folder}/results/depth*.png'))
        self.n_img = len(self.color_paths)
        self.poses = load_replica_poses(f'{self.input_folder}/traj.txt', self.n_img)


def _flip_pose(c2w):
    """float64 [4,4] c2w in the dataset's camera axes -> the codebase's (columns 1 and 2
    negated), as a float32 tensor."""
    c2w[:3, 1] *= -1
    c2w[:3, 2] *= -1
    return torch.from_numpy(c2w).float()


def _identity_poses(n):
    return [torch.from_numpy(np.eye(4)).float() for _ in range(n)]


class Azure(BaseDataset):
    """datasets.py:336-370: color/*.jpg and depth/*.png in lexicographic order; scene/trajectory.log
    in 5-line blocks (a header line, then four rows of the c2w), or the identity for every frame
    when that file is missing."""

    def __init__(self, data_path, device='cuda:0'):
        super().__init__(data_path, device)
        self.color_paths = sorted(glob.glob(os.path.join(self.input_folder, 'color', '*.jpg')))
        self.depth_paths = sorted(glob.glob(os.path.join(self.input_folder, 'depth', '*.png')))
        self.n_img = len(self.color_paths)
        self.poses = self.load_poses(os.path.join(self.input_folder, 'scene', 'trajectory.log'))

    def load_poses(self, path):
        if not os.path.exists(path):
            return _identity_poses(self.n_img)
        with open(path) as f:
            content = f.readlines()
        poses = []
        for i in range(0, len(content), 5):
            rows = ''.join(content[i + 1:i + 5]).strip().split()
            poses.append(_flip_pose(np.array(list(map(float, rows))).reshape((4, 4))))
        return poses


def _int_stem(path):
    """ScanNet's sort key: the integer before the 4-character extension."""
    return int(os.path.basename(path)[:-4])


class ScanNet(BaseDataset):
    """datasets.py:373-401: devices.yaml in the data root, frames under frames/: color/*.jpg,
    depth/*.png and pose/*.txt, each sorted by the integer file stem; pose rows split on single
    spaces (non-finite poses, as ScanNet has for lost frames, pass through)."""

    def __init__(self, data_path, device='cuda:0'):
        super().__init__(data_path, device)
        self.input_folder = os.path.join(self.input_folder, 'frames')
        self.color_paths = sorted(glob.glob(os.path.join(self.input_folder, 'color', '*.jpg')),
                                  key=_int_stem)
        self.depth_paths = sorted(glob.glob(os.path.join(self.input_folder, 'depth', '*.png')),
                                  key=_int_stem)
        self.poses = self.load_poses(os.path.join(self.input_folder, 'pose'))
        self.n_img = len(self.color_paths)

    def load_poses(self, path):
        poses = []
        for pose_path in sorted(glob.glob(os.path.join(path, '*.txt')), key=_int_stem):
            with open(pose_path) as f:
                vals = [list(map(float, line.split(' '))) for line in f.readlines()]
            poses.append(_flip_pose(np.array(vals).reshape(4, 4)))
        return poses


def _scenes7_key(path):
    """7-Scenes' sort key: the integer after the last '-' of the name's first dot-field
    (frame-000012.color.png -> 12)."""
    return int(os.path.basename(path).split('.')[0].split('-')[-1])


class Scenes7(BaseDataset):
    """datasets.py:404-435: *.color.png, *.depth.png and *.txt poses in one folder, sorted by
    frame number; pose rows are tab-separated."""

    def __init__(self, data_path, device='cuda:0'):
        super().__init__(data_path, device)
        self.color_paths = sorted(glob.glob(os.path.join(self.input_folder, '*.color.png')),
                                  key=_scenes7_key)
        self.depth_paths = sorted(glob.glob(os.path.join(self.input_folder, '*.depth.png')),
                                  key=_scenes7_key)
        self.poses = self.load_poses(self.input_folder)
        self.n_img = len(self.color_paths)

    def load_poses(self, path):
        poses = []
        for pose_path in sorted(glob.glob(os.path.join(path, '*.txt')), key=_scenes7_key):
            with open(pose_path) as f:
                vals = [list(map(float, line.strip().split('\t'))) for line in f.readlines()]
            poses.append(_flip_pose(np.array(vals).reshape(4, 4)))
        return poses


class CoFusion(BaseDataset):
    """datasets.py:438-458: colour/*.png and float32 OpenEXR depth_noise/*.exr.  Every pose is
    the identity: the reference could not align CoFusion's trajectories with the codebase's
    frame, and ATE aligns the trajectories anyway."""

    def __init__(self, data_path, device='cuda:0'):
        super().__init__(data_path, device)
        self.color_paths = sorted(glob.glob(os.path.join(self.input_folder, 'colour', '*.png')))
        self.depth_paths = sorted(glob.glob(os.path.join(self.input_folder, 'depth_noise',
                                                         '*.exr')))
        self.n_img = len(self.color_paths)
        self.poses = _identity_poses(self.n_img)


def tum_parse_list(filepath, skiprows=0):
    """datasets.py:468-474: a space-separated list file as strings ('#' lines skipped)."""
    import warnings
    with warnings.catch_warnings():
        # numpy notes that '#' lines do not count towards max_rows; nothing here sets it
        warnings.filterwarnings('ignore', 'Input line', UserWarning)
        return np.loadtxt(filepath, delimiter=' ', dtype=np.str_, skiprows=skiprows)


def tum_associate(tstamp_image, tstamp_depth, tstamp_pose, max_dt=0.08):
    """datasets.py:476-497: (image, depth, pose) index triples, each image paired with the
    nearest depth and the nearest pose (argmin |dt|, first on ties), kept when both are closer
    than max_dt seconds."""
    associations = []
    for i, t in enumerate(tstamp_image):
        j = np.argmin(np.abs(tstamp_depth - t))
        k = np.argmin(np.abs(tstamp_pose - t))
        if (np.abs(tstamp_depth[j] - t) < max_dt) and (np.abs(tstamp_pose[k] - t) < max_dt):
            associations.append((i, j, k))
    return associations


def tum_pose_matrix(pvec):
    """datasets.py:546-553: tx ty tz qx qy qz qw -> float64 [4,4]."""
    from scipy.spatial.transform import Rotation
    pose = np.eye(4)
    pose[:3, :3] = Rotation.from_quat(pvec[3:]).as_matrix()
    pose[:3, 3] = pvec[:3]
    return pose


def load_tum(datapath, frame_rate=-1):
    """datasets.py:499-544: -> (colour paths, depth paths, float32 c2w tensors).

    The pose list is groundtruth.txt, else pose.txt, read with skiprows=1 as the reference does
    (so a pose.txt without a header loses its first row).  Associated frames are subsampled:
    an image is kept when it is more than 1 / frame_rate seconds after the last kept one."""
    pose_list = None
    for name in ('groundtruth.txt', 'pose.txt'):
        if os.path.isfile(os.path.join(datapath, name)):
            pose_list = os.path.join(datapath, name)
            break
    if pose_list is None:
        raise FileNotFoundError(f'{datapath}: a TUM RGB-D folder needs groundtruth.txt or '
                                'pose.txt')
    image_data = tum_parse_list(os.path.join(datapath, 'rgb.txt'))
    depth_data = tum_parse_list(os.path.join(datapath, 'depth.txt'))
    pose_data = tum_parse_list(pose_list, skiprows=1)
    pose_vecs = pose_data[:, 1:].astype(np.float64)
    tstamp_image = image_data[:, 0].astype(np.float64)
    tstamp_depth = depth_data[:, 0].astype(np.float64)
    tstamp_pose = pose_data[:, 0].astype(np.float64)
    associations = tum_associate(tstamp_image, tstamp_depth, tstamp_pose)
    if not associations:
        raise ValueError(f'{datapath}: no image has a depth image and a pose within 0.08 s')
    indices = [0]
    for i in range(1, len(associations)):
        t0 = tstamp_image[associations[indices[-1]][0]]
        t1 = tstamp_image[associations[i][0]]
        if t1 - t0 > 1.0 / frame_rate:
            indices += [i]
    images, depths, poses = [], [], []
    for ix in indices:
        i, j, k = associations[ix]
        images.append(os.path.join(datapath, image_data[i, 1]))
        depths.append(os.path.join(datapath, depth_data[j, 1]))
        poses.append(_flip_pose(tum_pose_matrix(pose_vecs[k])))
    return images, depths, poses


class TUM_RGBD(BaseDataset):
    """datasets.py:461-553: rgb.txt / depth.txt / groundtruth.txt (or pose.txt) associated by
    timestamp and subsampled at 32 frames per second (`load_tum`)."""

    def __init__(self, data_path, device='cuda:0'):
        super().__init__(data_path, device)
        self.color_paths, self.depth_paths, self.poses = load_tum(self.input_folder,
                                                                  frame_rate=32)
        self.n_img = len(self.color_paths)


# datasets.py:556-564 without 'euroc' (get_dataset explains why)
dataset_dict = {
    'replica': Replica,
    'scannet': ScanNet,
    'cofusion': CoFusion,
    'azure': Azure,
    'tumrgbd': TUM_RGBD,
    '7scenes': Scenes7,
}
