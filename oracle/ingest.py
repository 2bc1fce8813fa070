"""numpy restatement of csrc/ingest.cu (test infrastructure only, never on the product path).

The frame transform of a Replica-style RGB-D folder (slam/common/datasets.py:95-134, the
reference's BaseDataset.__getitem__), written as the kernel computes it:

  1. undistort (colour only, uint8, when distortion coefficients are given): cv::undistort's model
     -- initUndistortRectifyMap with new camera matrix = K in 4096-pixel row stripes, CV_16SC2
     maps with 1/32-pixel fractions, remap INTER_LINEAR with 15-bit fixed-point weights and
     BORDER_CONSTANT 0;
  2. BGR -> RGB and `/ 255.` in float64;
  3. depth = float32(u16) / float32(png_depth_scale) in float32;
  4. colour resized to the depth's size (cv2.resize INTER_LINEAR on float64: float32 coefficients,
     a copy when the sizes match);
  5. crop of `crop_edge` pixels on every side;
  6. downsample to ((H-2e)//f, (W-2e)//f) when f > 1: colour INTER_LINEAR on float64 (cv2's
     2x2 area average when the scale is exactly 2 on both axes), depth INTER_NEAREST;
  7. colour cast to float32.

numpy's float32 / float64 elementwise operations round to nearest and are never contracted, so
writing the kernel's expressions in the same order reproduces it bit for bit.

One deliberate difference from cv2's own loop: the undistortion map's column coordinate is
ir[2] + j * ir[0] per pixel, where initUndistortRectifyMap accumulates _x += ir[0] along the row
(or, in its SIMD path, adds lane offsets with fused multiply-adds).  The three agree to ~1e-15
pixel before the map is rounded to 1/32 pixel, so they give the same map except where u * 32
lies within that distance of a rounding boundary; tests/golden/ingest_ref.npz (real cv2) pins
that no recorded case meets one."""
from __future__ import annotations

import numpy as np

f32, f64 = np.float32, np.float64
INTER_BITS = 5
INTER_TAB = 1 << INTER_BITS        # 32 map fractions per pixel
COEF_BITS = 15                     # remap's fixed-point weight scale 2^15
STRIPE_PIXELS = 1 << 12            # cv::undistort processes rows in stripes of 4096 / W rows


def output_size(h, w, crop_edge, downsample_factor):
    """(h, w) of the frames the transform produces from a (h, w) depth image."""
    h, w = h - 2 * crop_edge, w - 2 * crop_edge
    if downsample_factor > 1:
        h, w = h // downsample_factor, w // downsample_factor
    return h, w


def dist_coeffs(dist):
    """k1 k2 p1 p2 k3 k4 k5 k6 s1 s2 s3 s4 (float64), zero-filled from 4, 5, 8 or 12 values."""
    d = np.zeros(12, f64)
    dist = np.asarray(dist, f64).ravel()
    if dist.size not in (4, 5, 8, 12):
        raise ValueError(f'{dist.size} distortion coefficients (4, 5, 8 or 12 are supported)')
    d[:dist.size] = dist
    return d


def undistort_map(H, W, fx, fy, cx, cy, dist):
    """-> (sx, sy) int32 [H,W] integer source pixel and frac int32 [H,W] = fy32 * 32 + fx32."""
    k1, k2, p1, p2, k3, k4, k5, k6, s1, s2, s3, s4 = (f64(v) for v in dist_coeffs(dist))
    fx, fy, cx, cy = f64(fx), f64(fy), f64(cx), f64(cy)
    stripe = min(max(1, STRIPE_PIXELS // max(W, 1)), H)
    rows = np.arange(H)
    y0 = (rows // stripe) * stripe
    i = (rows - y0).astype(f64)[:, None]
    cyp = (cy - y0.astype(f64))[:, None]          # Ar(1,2) = v0 - y of the stripe
    # (Ar)^-1 by cv::invert's 3x3 cofactor formula: d = 1 / det, t = cofactor * d
    d = f64(1.0) / (fx * fy)
    ir0 = fy * d
    ir2 = (f64(0.0) - cx * fy) * d
    ir4 = fx * d
    ir5 = (f64(0.0) - fx * cyp) * d
    ir8 = (fx * fy) * d
    j = np.arange(W, dtype=f64)[None, :]
    _x = ir2 + j * ir0
    _y = i * ir4 + ir5
    w = f64(1.0) / ir8
    x = _x * w
    y = _y * w
    x2 = x * x
    y2 = y * y
    r2 = x2 + y2
    _2xy = f64(2.0) * x * y
    kr = ((f64(1.0) + ((k3 * r2 + k2) * r2 + k1) * r2) /
          (f64(1.0) + ((k6 * r2 + k5) * r2 + k4) * r2))
    xd = x * kr + p1 * _2xy + p2 * (r2 + f64(2.0) * x2) + s1 * r2 + s2 * r2 * r2
    yd = y * kr + p1 * (r2 + f64(2.0) * y2) + p2 * _2xy + s3 * r2 + s4 * r2 * r2
    u = fx * xd + cx
    v = fy * yd + cy
    iu = np.rint(u * f64(INTER_TAB)).astype(np.int64)   # cvRound: half to even
    iv = np.rint(v * f64(INTER_TAB)).astype(np.int64)
    sx = (iu >> INTER_BITS).astype(np.int32)
    sy = (iv >> INTER_BITS).astype(np.int32)
    frac = ((iv & (INTER_TAB - 1)) * INTER_TAB + (iu & (INTER_TAB - 1))).astype(np.int32)
    return sx, sy, frac


def remap_bilinear_u8(img, sx, sy, frac):
    """remap INTER_LINEAR of a uint8 [H0,W0,C] image through a CV_16SC2 + CV_16UC1 map pair,
    BORDER_CONSTANT 0: sum of the four corners' values (0 outside) times their 15-bit weights,
    (sum + 2^14) >> 15."""
    H0, W0, C = img.shape
    ax = (frac & (INTER_TAB - 1)).astype(np.int64)
    ay = (frac >> INTER_BITS).astype(np.int64)
    # bilinear table entry: products of k/32 fractions scaled by 2^15 are exact integers
    wts = [(INTER_TAB - ax) * (INTER_TAB - ay) * INTER_TAB, ax * (INTER_TAB - ay) * INTER_TAB,
           (INTER_TAB - ax) * ay * INTER_TAB, ax * ay * INTER_TAB]
    acc = np.zeros(sx.shape + (C,), np.int64)
    for k, (dx, dy) in enumerate(((0, 0), (1, 0), (0, 1), (1, 1))):
        x, y = sx.astype(np.int64) + dx, sy.astype(np.int64) + dy
        inside = (x >= 0) & (x < W0) & (y >= 0) & (y < H0)
        v = img[np.clip(y, 0, H0 - 1), np.clip(x, 0, W0 - 1)].astype(np.int64)
        acc += np.where(inside[..., None], v, 0) * wts[k][..., None]
    return np.clip((acc + (1 << (COEF_BITS - 1))) >> COEF_BITS, 0, 255).astype(np.uint8)


def undistort(img, fx, fy, cx, cy, dist):
    H, W = img.shape[:2]
    return remap_bilinear_u8(img, *undistort_map(H, W, fx, fy, cx, cy, dist))


def _scale(src, dst):
    """cv::resize's scale: 1 / (dst / src) in double."""
    return f64(1.0) / (f64(dst) / f64(src))


def linear_coeffs(src, dst, clamp):
    """Source index and float32 weights (1 - t, t) of each destination index of an INTER_LINEAR
    resize.  t = float32((d + 0.5) * scale - 0.5) - floor.  Along x (clamp=True) an index below 0
    or at/after src - 1 is clamped with weight (1, 0); along y the index is not clamped (the rows
    are, when they are fetched)."""
    scale = _scale(src, dst)
    t = ((np.arange(dst, dtype=f64) + f64(0.5)) * scale - f64(0.5)).astype(f32)
    s = np.floor(t).astype(np.int64)
    t = (t - s.astype(f32)).astype(f32)
    if clamp:
        low = s < 0
        t[low], s[low] = f32(0), 0
        high = s >= src - 1
        t[high], s[high] = f32(0), src - 1
    return s, (f32(1) - t).astype(f32), t


def is_area2(sh, sw, dh, dw):
    """cv2.resize turns INTER_LINEAR into its fast 2x2 area average when both scales are 2."""
    eps = np.finfo(f64).eps
    sx, sy = _scale(sw, dw), _scale(sh, dh)
    return abs(sx - 2.0) < eps and abs(sy - 2.0) < eps


def resize_linear_f64(img, dh, dw):
    """cv2.resize(img, (dw, dh)) (INTER_LINEAR) of a float64 [h,w,C] image."""
    sh, sw = img.shape[:2]
    img = np.asarray(img, f64)
    if (sh, sw) == (dh, dw):
        return img.copy()
    if is_area2(sh, sw, dh, dw):
        s00, s01 = img[0:2 * dh:2, 0:2 * dw:2], img[0:2 * dh:2, 1:2 * dw:2]
        s10, s11 = img[1:2 * dh:2, 0:2 * dw:2], img[1:2 * dh:2, 1:2 * dw:2]
        return (f64(0.0) + s00 + s01 + s10 + s11) * f64(f32(0.25))
    xs, xa0, xa1 = linear_coeffs(sw, dw, True)
    ys, yb0, yb1 = linear_coeffs(sh, dh, False)
    xs1 = np.minimum(xs + 1, sw - 1)   # weight 0 wherever xs + 1 is out of range
    hrow = img[:, xs] * xa0.astype(f64)[None, :, None] + img[:, xs1] * xa1.astype(f64)[None, :, None]
    r0 = np.clip(ys, 0, sh - 1)
    r1 = np.clip(ys + 1, 0, sh - 1)
    return hrow[r0] * yb0.astype(f64)[:, None, None] + hrow[r1] * yb1.astype(f64)[:, None, None]


def resize_nearest(img, dh, dw):
    """cv2.resize(img, (dw, dh), interpolation=INTER_NEAREST): floor(d * (1 / (dst / src)))."""
    sh, sw = img.shape[:2]
    if (sh, sw) == (dh, dw):
        return img.copy()
    ix = np.minimum(np.floor(np.arange(dw, dtype=f64) * _scale(sw, dw)).astype(np.int64), sw - 1)
    iy = np.minimum(np.floor(np.arange(dh, dtype=f64) * _scale(sh, dh)).astype(np.int64), sh - 1)
    return img[iy][:, ix]


def ingest(color_bgr, depth_u16, fx, fy, cx, cy, dist=None, png_depth_scale=6553.5, crop_edge=0,
           downsample_factor=1):
    """One frame: uint8 BGR [H0,W0,3] and uint16 [Hd,Wd] -> (rgb f32 [h,w,3], depth f32 [h,w])."""
    color = np.asarray(color_bgr, np.uint8)
    if dist is not None:
        color = undistort(color, fx, fy, cx, cy, dist)
    color = color[..., ::-1].astype(f64) / f64(255.0)
    depth = np.asarray(depth_u16, np.uint16).astype(f32) / f32(png_depth_scale)
    Hd, Wd = depth.shape
    color = resize_linear_f64(color, Hd, Wd)
    e = crop_edge
    if e > 0:
        color, depth = color[e:-e, e:-e], depth[e:-e, e:-e]
    if downsample_factor > 1:
        h, w = output_size(Hd, Wd, e, downsample_factor)
        color = resize_linear_f64(color, h, w)
        depth = resize_nearest(depth, h, w)
    return color.astype(f32), np.ascontiguousarray(depth, f32)
