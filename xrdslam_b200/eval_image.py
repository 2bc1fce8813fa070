"""Render-quality metrics of re-rendered frames on the device (csrc/eval_image.cu): the PSNR,
MS-SSIM and rendered-depth L1 that save_render_imgs reports (slam/common/common.py:429-479,
reference @ f0366f20), batched over frames.  Semantics in include/xrdslam_b200.h under
xrd_eval_image_*.

LPIPS needs AlexNet and the LPIPS linear-layer weights, which this package does not ship: it
comes from an optional `lpips_fn(gt, pred) -> float` hook and is NaN without one.  The
reference's matplotlib figures are not written."""
from __future__ import annotations

import numpy as np
import torch

from . import _cabi
from ._cabi import (XRD_EVAL_IMAGE_MAX_SIDE, XRD_EVAL_IMAGE_MIN_SIDE, XRD_EVAL_IMAGE_NO_DEPTH,
                    XRD_EVAL_IMAGE_OUT, ptr)

PSNR, SSIM, DEPTH_L1, MSE = range(XRD_EVAL_IMAGE_OUT)


def _device(device=None):
    dev = torch.device(device if device is not None else 'cuda:0')
    _cabi.require_cuda(dev, 'the render metrics')
    return dev


def _tensor(x, dev, dtype):
    t = torch.from_numpy(np.ascontiguousarray(x)) if isinstance(x, np.ndarray) else \
        torch.as_tensor(x)
    return t.to(dev, dtype).contiguous()


def image_metrics(gt_color, gt_depth, color, depth=None, out=None, levels=None):
    """xrd_eval_image_metrics on DEVICE tensors: gt_color, color f32 [B,H,W,3], gt_depth f32
    [B,H,W], depth f64 [B,H,W] or None (no rendered depth: the colours are masked by
    gt_depth > 0 and depth_l1 is 0).  -> out DEVICE f64 [B,4] = (psnr, ms_ssim, depth_l1, mse),
    enqueued on the current stream with no host synchronisation.  levels: a DEVICE f64
    [B,5,3,2] to receive the per-level (mean ssim, mean cs), or None."""
    dev = gt_depth.device
    gt_color = gt_color.to(dev, torch.float32).contiguous()
    color = color.to(dev, torch.float32).contiguous()
    gt_depth = gt_depth.to(torch.float32).contiguous()
    if depth is not None:
        depth = depth.to(dev, torch.float64).contiguous()
    if gt_depth.dim() != 3:
        raise ValueError(f'gt_depth must be [B,H,W], got {tuple(gt_depth.shape)}')
    B, H, W = gt_depth.shape
    for name, t, shape in (('gt_color', gt_color, (B, H, W, 3)), ('color', color, (B, H, W, 3)),
                           ('depth', depth, (B, H, W))):
        if t is not None and tuple(t.shape) != shape:
            raise ValueError(f'{name} must be {list(shape)}, got {list(t.shape)}')
    if min(H, W) < XRD_EVAL_IMAGE_MIN_SIDE or max(H, W) > XRD_EVAL_IMAGE_MAX_SIDE:
        raise ValueError(f'MS-SSIM needs both image sides > (11 - 1) * 2**4 = 160 (and at most '
                         f'{XRD_EVAL_IMAGE_MAX_SIDE}), got {H} x {W}')
    if out is None:
        out = torch.empty(B, XRD_EVAL_IMAGE_OUT, dtype=torch.float64, device=dev)
    ws, nb = _cabi.workspace(
        dev, 'eval_image', B, H, W,
        error=f'render metrics: unsupported batch of {B} frames of {H} x {W}')
    flags = XRD_EVAL_IMAGE_NO_DEPTH if depth is None else 0
    _cabi.launch_on(dev, 'xrd_eval_image_metrics', ptr(gt_color), ptr(color), ptr(gt_depth),
                    ptr(depth), B, H, W, flags, ptr(out), ptr(levels), ptr(ws), nb)
    return out


def lpips_inputs(gt_color, color, gt_depth, masked):
    """The colours save_render_imgs gives LPIPS: both clipped to [0, 1] and, without a rendered
    depth, multiplied by gt_depth > 0."""
    a, v = gt_color.clamp(0, 1), color.clamp(0, 1)
    if masked:
        m = (gt_depth > 0).unsqueeze(-1).to(a.dtype)
        a, v = a * m, v * m
    return a, v


def render_metrics(gt_color, gt_depth, color, depth, lpips_fn=None, device=None):
    """The metrics of save_render_imgs for one frame ([H,W,3] / [H,W]) or a batch ([B,H,W,3] /
    [B,H,W]) of numpy arrays or tensors: gt_color, color, gt_depth and the rendered depth (or
    None: the colours are masked by gt_depth > 0 and depth_l1 is 0).  -> None when color is None,
    else {'psnr', 'ssim', 'lpips', 'depth_l1'}: floats for one frame, f64 arrays [B] for a
    batch.  LPIPS is lpips_fn(gt, pred) of the clipped (masked) DEVICE colours [H,W,3], called
    once per frame, or NaN without the hook.  One host read."""
    if color is None:
        return None
    if device is None:
        device = next((t.device for t in (gt_color, color, gt_depth, depth)
                       if torch.is_tensor(t) and t.is_cuda), None)
    dev = _device(device)
    single = np.ndim(gt_depth) == 2
    gc = _tensor(gt_color, dev, torch.float32)
    c = _tensor(color, dev, torch.float32)
    gd = _tensor(gt_depth, dev, torch.float32)
    d = None if depth is None else _tensor(depth, dev, torch.float64)
    if single:
        gc, c, gd = gc[None], c[None], gd[None]
        d = None if d is None else d[None]
    out = image_metrics(gc, gd, c, d)
    lp = [float('nan')] * gd.shape[0]
    if lpips_fn is not None:
        for k in range(gd.shape[0]):
            lp[k] = lpips_fn(*lpips_inputs(gc[k], c[k], gd[k], d is None))
    o = out.cpu().numpy()
    res = {'psnr': o[:, PSNR], 'ssim': o[:, SSIM], 'lpips': np.array([float(v) for v in lp]),
           'depth_l1': o[:, DEPTH_L1]}
    return {k: float(v[0]) for k, v in res.items()} if single else res
