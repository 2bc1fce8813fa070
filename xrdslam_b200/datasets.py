"""RGB-D dataset readers (slam/common/datasets.py): the Replica folder layout, decoded on the host
and turned into float32 device frames by one CUDA call (csrc/ingest.cu, `frame_ingest`).

`dataset[i]` returns `(i, rgb f32 [h,w,3], depth f32 [h,w], c2w f32 [4,4])` as device tensors,
the protocol of the reference's BaseDataset.__getitem__ (datasets.py:95-134).  The colour is
undistorted, converted, resized, cropped and downsampled exactly as that method does with cv2
(see include/xrdslam_b200.h, xrd_frame_ingest).

Decoding uses cv2.imread when cv2 is importable, as the reference does; otherwise PIL, whose
JPEG decoder may round differently from cv2's libjpeg build, so the pixels then match the
reference's only up to the decoder.  `DECODER` names the one in use.

Iterating a dataset in order prefetches: a host thread decodes frame i + 1 into pinned memory
while frame i is being used (the reference's DataLoader(num_workers=1), without its float64 host
work).  Only the Replica layout is read here; other layouts differ in file listing and pose
parsing and can reuse `frame_ingest`."""
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

    color: uint8 [B,H0,W0,3] (BGR, cv2.imread's order); depth: uint16 or int16 (same bits)
    [B,Hd,Wd].  One or two launches on the current stream, no host synchronisation.  `out` may
    hold preallocated (rgb, depth) tensors."""
    from . import _cabi
    if color.dim() == 3:
        color, depth = color[None], depth[None]
    if color.dtype != torch.uint8 or depth.dtype not in (torch.int16, torch.uint16):
        raise TypeError('frame_ingest needs uint8 colour and 16-bit depth')
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
    _cabi.launch_on(dev, 'xrd_frame_ingest', cfg, _cabi.ptr(color), _cabi.ptr(depth),
                    _cabi.ptr(rgb), _cabi.ptr(dep), _cabi.ptr(ws), nbytes)
    return rgb, dep


def get_dataset(data_path, data_type, device='cuda:0'):
    return dataset_dict[data_type](data_path, device=device)


def load_config(path):
    import yaml
    with open(path) as f:
        return yaml.safe_load(f)


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
        holding the uint16 depth bits)."""
        color = read_color(self.color_paths[index])
        depth = read_depth(self.depth_paths[index]).view(np.int16)
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


dataset_dict = {'replica': Replica}
