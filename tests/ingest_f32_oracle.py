"""The frame transform with float32 (OpenEXR) depth, composed from oracle/ingest.py's stages:
colour exactly as oracle.ingest.ingest, depth = float32(d) / float32(png_depth_scale) in numpy
(x86 division: IEEE, NaN payloads kept), cropped, then INTER_NEAREST when downsampling."""
import numpy as np

from oracle import ingest as O


def ingest_f32(color_bgr, depth_f32, fx, fy, cx, cy, dist=None, png_depth_scale=1.0,
               crop_edge=0, downsample_factor=1):
    """One frame: uint8 BGR [H0,W0,3] and float32 [Hd,Wd] -> (rgb f32 [h,w,3], depth f32 [h,w])."""
    depth = np.asarray(depth_f32, np.float32)
    rgb, _ = O.ingest(color_bgr, np.zeros(depth.shape, np.uint16), fx, fy, cx, cy, dist,
                      png_depth_scale, crop_edge, downsample_factor)
    with np.errstate(invalid='ignore', divide='ignore', over='ignore', under='ignore'):
        depth = depth.astype(np.float32) / np.float32(png_depth_scale)
    Hd, Wd = depth.shape
    e = crop_edge
    if e > 0:
        depth = depth[e:-e, e:-e]
    if downsample_factor > 1:
        depth = O.resize_nearest(depth, *O.output_size(Hd, Wd, e, downsample_factor))
    return rgb, np.ascontiguousarray(depth, np.float32)
