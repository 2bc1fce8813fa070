"""Restatements of the render-quality metrics (test infrastructure only, never on the product
path):

(a) `metrics`: csrc/eval_image.cu in numpy, in the kernels' operation order -- fp32 window,
    filter and SSIM maps, the same 2x2 pooling order and the same fixed-order f64 partial sums --
    so the device results are reproduced bit for bit (log10 and pow aside, see `metrics`).
(b) `save_render_imgs` / `ms_ssim`: the reference's metric code (slam/common/common.py:429-479,
    reference @ f0366f20) in torch, with pytorch_msssim.ms_ssim restated from memory (the library
    is not installed: parity with it is unpinned) on F.conv2d(groups=C) and F.avg_pool2d, fed the
    reference's transpose(0, 2) layout.  It stands for the reference's semantics.

numpy's float32 / float64 elementwise operations round to nearest and are never contracted, so
writing the kernels' expressions in the same order reproduces them."""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

f32, f64 = np.float32, np.float64
WIN = 11
TILE_W, TILE_H, THREADS, CHUNK = 32, 16, 256, 4096
LEVELS = 5
C1, C2 = f32(0.01 * 0.01), f32(0.03 * 0.03)
WEIGHTS = (0.0448, 0.2856, 0.3001, 0.2363, 0.1333)


# ---------------------------------------------------------------- (a) the kernels' arithmetic ---
def window():
    """f32 [11]: g_k = fp32(exp(fp32(-(d d) / 4.5))), d = k - 5, over its in-order fp32 sum."""
    d = (np.arange(WIN) - WIN // 2).astype(f32)
    q = -(d * d) / f32(4.5)
    g = np.array([math.exp(float(v)) for v in q]).astype(f32)
    s = f32(0)
    for v in g:
        s = f32(s + v)
    return g / s


def _tree(a):
    """The kernels' fixed tree over the last axis (256 thread values)."""
    h = a.shape[-1] // 2
    while h:
        a = a[..., :h] + a[..., h:2 * h]
        h //= 2
    return a[..., 0]


def fixed_sum(v):
    """f64 [..., n] -> [...]: thread t of 256 sums elements t, t + 256, ... in order, then the
    tree."""
    n = v.shape[-1]
    m = max(1, -(-n // THREADS))
    p = np.zeros(v.shape[:-1] + (m * THREADS, ), f64)
    p[..., :n] = v
    p = p.reshape(v.shape[:-1] + (m, THREADS))
    acc = np.zeros(v.shape[:-1] + (THREADS, ), f64)
    for r in range(m):
        acc = acc + p[..., r, :]
    return _tree(acc)


def _clip(v):
    return np.minimum(np.maximum(np.asarray(v, f32), f32(0)), f32(1))


def colors(gt_color, color, gt_depth, mask):
    """The level-0 colours: clipped, and masked by gt_depth > 0 when `mask`."""
    a, v = _clip(gt_color), _clip(color)
    if mask:
        m = (np.asarray(gt_depth) > 0).astype(f32)[..., None]
        a, v = a * m, v * m
    return a, v


def frame_sums(a, v, gt_depth, depth):
    """[B,H,W,3] colours (already clipped / masked), gt f32 [B,H,W], depth f64 [B,H,W] or None
    -> f64 [B,3] = (sum of squared errors, sum |gt - r| over gt > 0, count)."""
    B, H, W, _ = a.shape
    n = H * W
    nch = -(-n // CHUNK)

    def chunked(e):   # [B, n, k] per-pixel terms -> per-chunk partials [B, nch]
        k = e.shape[-1]
        p = np.zeros((B, nch * CHUNK, k), f64)
        p[:, :n] = e
        p = p.reshape(B, nch, CHUNK // THREADS, THREADS, k)
        acc = np.zeros((B, nch, THREADS), f64)
        for i in range(CHUNK // THREADS):
            for c in range(k):
                acc = acc + p[:, :, i, :, c]
        return fixed_sum(_tree(acc))

    d = a - v
    se = chunked((d * d).astype(f64).reshape(B, n, 3))
    if depth is None:
        return np.stack([se, np.zeros(B), np.zeros(B)], -1)
    g = np.asarray(gt_depth, f32).reshape(B, n)
    ok = g > 0
    dl = np.where(ok, np.abs(g.astype(f64) - np.asarray(depth, f64).reshape(B, n)), 0.0)
    return np.stack([se, chunked(dl[..., None]), chunked(ok.astype(f64)[..., None])], -1)


def _filter(img, w):
    """Valid 11-tap correlation along x, then along y; f32, taps summed in order."""
    H, W = img.shape[-2:]
    h = np.zeros(img.shape[:-1] + (W - WIN + 1, ), f32)
    for k in range(WIN):
        h = h + w[k] * img[..., k:k + W - WIN + 1]
    o = np.zeros(img.shape[:-2] + (H - WIN + 1, W - WIN + 1), f32)
    for k in range(WIN):
        o = o + w[k] * h[..., k:k + H - WIN + 1, :]
    return o


def _tile_sums(m):
    """f32 map [B,3,Ho,Wo] -> f64 [B,3]: per 32 x 16 tile, thread (r, q) adds rows r and r + 8 of
    column q, the tree, then the tile sums in tile order."""
    B, C, Ho, Wo = m.shape
    ty, tx = -(-Ho // TILE_H), -(-Wo // TILE_W)
    p = np.zeros((B, C, ty * TILE_H, tx * TILE_W), f64)
    p[:, :, :Ho, :Wo] = m
    p = p.reshape(B, C, ty, 2, TILE_H // 2, tx, TILE_W).transpose(0, 1, 2, 5, 3, 4, 6)
    acc = (0.0 + p[..., 0, :, :]) + p[..., 1, :, :]            # [B,C,ty,tx,8,32]
    per_tile = _tree(acc.reshape(B, C, ty * tx, THREADS))
    return fixed_sum(per_tile)


def ssim_level(x, y, w):
    """Planar f32 [B,3,H,W] -> (mean ssim, mean cs) f64 [B,3] each."""
    mu1, mu2 = _filter(x, w), _filter(y, w)
    exx, eyy, exy = _filter(x * x, w), _filter(y * y, w), _filter(x * y, w)
    mu1_sq, mu2_sq, mu12 = mu1 * mu1, mu2 * mu2, mu1 * mu2
    s1, s2, s12 = exx - mu1_sq, eyy - mu2_sq, exy - mu12
    cs = (f32(2) * s12 + C2) / ((s1 + s2) + C2)
    ssim = ((f32(2) * mu12 + C1) / ((mu1_sq + mu2_sq) + C1)) * cs
    n = float(cs.shape[-2]) * float(cs.shape[-1])
    return _tile_sums(ssim) / n, _tile_sums(cs) / n


def pool(x):
    """avg_pool2d(2, 2, padding s % 2, count_include_pad) of planar f32 [B,3,H,W], the window
    summed row by row."""
    B, C, H, W = x.shape
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    p = np.zeros((B, C, 2 * Ho, 2 * Wo), f32)
    p[:, :, H % 2:H % 2 + H, W % 2:W % 2 + W] = x
    p = p.reshape(B, C, Ho, 2, Wo, 2)
    s = ((p[:, :, :, 0, :, 0] + p[:, :, :, 0, :, 1]) + p[:, :, :, 1, :, 0]) + p[:, :, :, 1, :, 1]
    return s * f32(0.25)


def metrics(gt_color, gt_depth, color, depth=None):
    """xrd_eval_image_metrics in numpy: [B,H,W,3] / [B,H,W] inputs, depth None = no rendered
    depth (colours masked) -> (out f64 [B,4] = psnr, ms_ssim, depth_l1, mse; levels f64
    [B,5,3,2] = mean ssim, mean cs).  Everything but psnr and ms_ssim is bit-exact; those two
    apply log10 / pow, which numpy and CUDA need not round alike."""
    a, v = colors(gt_color, color, gt_depth, depth is None)
    B, H, W, _ = a.shape
    fs = frame_sums(a, v, gt_depth, depth)
    w = window()
    x, y = a.transpose(0, 3, 1, 2), v.transpose(0, 3, 1, 2)
    levels = np.zeros((B, LEVELS, 3, 2))
    for lv in range(LEVELS):
        s, c = ssim_level(x, y, w)
        levels[:, lv, :, 0], levels[:, lv, :, 1] = s, c
        if lv + 1 < LEVELS:
            x, y = pool(x), pool(y)
    mse = fs[:, 0] / (3.0 * H * W)
    vals = np.maximum(levels[:, :, :, 1].copy(), 0.0)      # relu(cs), levels 0..3
    vals[:, -1] = np.maximum(levels[:, -1, :, 0], 0.0)     # relu(ssim), level 4
    wts = np.array(WEIGHTS, f32).astype(f64)
    p = vals[:, 0] ** wts[0]
    for lv in range(1, LEVELS):
        p = p * vals[:, lv] ** wts[lv]
    with np.errstate(divide='ignore', invalid='ignore'):
        out = np.stack([-10.0 * np.log10(mse), ((p[:, 0] + p[:, 1]) + p[:, 2]) / 3.0,
                        fs[:, 1] / fs[:, 2] * 100.0 if depth is not None else np.zeros(B),
                        mse], -1)
    return out, levels


# ---------------------------------------------------------------- (b) the reference in torch ---
def _fspecial_gauss_1d(size, sigma):
    coords = torch.arange(size, dtype=torch.float)
    coords -= size // 2
    g = torch.exp(-(coords ** 2) / (2 * sigma ** 2))
    g /= g.sum()
    return g.unsqueeze(0).unsqueeze(0)


def _gaussian_filter(x, win):
    C = x.shape[1]
    out = x
    for i, s in enumerate(x.shape[2:]):
        out = F.conv2d(out, weight=win.transpose(2 + i, -1), stride=1, padding=0, groups=C)
    return out


def _ssim(X, Y, data_range, win, K=(0.01, 0.03)):
    K1, K2 = K
    compensation = 1.0
    C1_, C2_ = (K1 * data_range) ** 2, (K2 * data_range) ** 2
    win = win.to(X.device, dtype=X.dtype)
    mu1, mu2 = _gaussian_filter(X, win), _gaussian_filter(Y, win)
    mu1_sq, mu2_sq, mu1_mu2 = mu1.pow(2), mu2.pow(2), mu1 * mu2
    sigma1_sq = compensation * (_gaussian_filter(X * X, win) - mu1_sq)
    sigma2_sq = compensation * (_gaussian_filter(Y * Y, win) - mu2_sq)
    sigma12 = compensation * (_gaussian_filter(X * Y, win) - mu1_mu2)
    cs_map = (2 * sigma12 + C2_) / (sigma1_sq + sigma2_sq + C2_)
    ssim_map = ((2 * mu1_mu2 + C1_) / (mu1_sq + mu2_sq + C1_)) * cs_map
    return torch.flatten(ssim_map, 2).mean(-1), torch.flatten(cs_map, 2).mean(-1)


def ms_ssim(X, Y, data_range=255, size_average=True, win_size=11, win_sigma=1.5, weights=None,
            K=(0.01, 0.03)):
    """pytorch_msssim.ms_ssim for 4-D inputs (restated from memory)."""
    smaller_side = min(X.shape[-2:])
    assert smaller_side > (win_size - 1) * (2 ** 4), \
        'Image size should be larger than %d due to the 4 downsamplings in ms-ssim' % (
            (win_size - 1) * (2 ** 4))
    if weights is None:
        weights = list(WEIGHTS)
    weights = X.new_tensor(weights)
    win = _fspecial_gauss_1d(win_size, win_sigma)
    win = win.repeat([X.shape[1]] + [1] * (len(X.shape) - 1))
    levels = weights.shape[0]
    mcs = []
    for i in range(levels):
        ssim_per_channel, cs = _ssim(X, Y, data_range=data_range, win=win, K=K)
        if i < levels - 1:
            mcs.append(torch.relu(cs))
            padding = [s % 2 for s in X.shape[2:]]
            X = F.avg_pool2d(X, kernel_size=2, padding=padding)
            Y = F.avg_pool2d(Y, kernel_size=2, padding=padding)
    ssim_per_channel = torch.relu(ssim_per_channel)
    mcs_and_ssim = torch.stack(mcs + [ssim_per_channel], dim=0)
    ms_ssim_val = torch.prod(mcs_and_ssim ** weights.view(-1, 1, 1), dim=0)
    return ms_ssim_val.mean() if size_average else ms_ssim_val.mean(1)


def save_render_imgs(gt_color_np, gt_depth_np, color_np, depth_np):
    """The metric part of common.py:429-479 -> (psnr, ssim, depth_l1_render) as Python floats,
    or None without a rendered colour (LPIPS and the figure are left out)."""
    gt_color_np = np.clip(gt_color_np, 0, 1)
    if color_np is None:
        return None
    color_np = np.clip(color_np, 0, 1)
    if depth_np is not None:
        gt_color, rcolor = torch.tensor(gt_color_np), torch.tensor(color_np)
        gt_depth, rdepth = torch.tensor(gt_depth_np), torch.tensor(depth_np)
        depth_l1_render = torch.abs(gt_depth[gt_depth_np > 0] - rdepth[gt_depth_np > 0]
                                    ).mean().item() * 100
    else:
        depth_mask = (torch.from_numpy(gt_depth_np > 0).unsqueeze(-1)).float()
        gt_color = torch.tensor(gt_color_np) * depth_mask
        rcolor = torch.tensor(color_np) * depth_mask
        depth_l1_render = 0.0
    mse_loss = F.mse_loss(gt_color, rcolor)
    psnr = -10. * torch.log10(mse_loss)
    ssim = ms_ssim(gt_color.transpose(0, 2).unsqueeze(0).float(),
                   rcolor.transpose(0, 2).unsqueeze(0).float(), data_range=1.0, size_average=True)
    return float(psnr), float(ssim), float(depth_l1_render)
