"""Render-quality metrics on the CPU: the numpy restatement of csrc/eval_image.cu (oracle (a))
against the torch restatement of the reference's save_render_imgs / pytorch_msssim.ms_ssim
(oracle (b)), analytic cases, and the host-side shape checks of the C-ABI."""
import numpy as np
import pytest
import torch

from oracle import eval_image as oe

f32 = np.float32
# Gates of (a) against (b), set a small factor above the maxima measured over the cases of
# test_kernel_order_against_reference_semantics (MS-SSIM 7.2e-6 absolute, PSNR 1.5e-7 relative,
# depth L1 2.3e-16 relative).  MS-SSIM: the fp32 E[x^2] - mu^2 cancellation is divided by
# denominators as small as C2, so fp32 summation order shows at 1e-5; PSNR: torch's mse is an
# fp32 mean, here it is an f64 sum.
SSIM_ABS = 2e-5
PSNR_REL = 5e-7
DEPTH_REL = 1e-12


def _synthetic(H, W, k=0):
    from xrdslam_b200.synthetic import make_sequence
    _, _, fr = make_sequence(k + 2, width=W, height=H)
    return fr[k][0], fr[k][1], fr[k + 1][0], fr[k + 1][1].astype(np.float64)


def _random(H, W, seed, noise=0.2):
    rng = np.random.default_rng(seed)
    g = rng.random((H, W, 3), dtype=f32)
    r = (g + rng.normal(0, noise, g.shape)).astype(f32)
    d = rng.random((H, W)).astype(f32) * 3
    d[d < 0.9] = 0
    return g, d, r, d + rng.normal(0, 0.05, d.shape)


def _a(gc, gd, c, d):
    out, _ = oe.metrics(gc[None], gd[None], c[None], None if d is None else d[None])
    return out[0]


def _check_against_b(gc, gd, c, d):
    psnr, ssim, dl1 = oe.save_render_imgs(gc, gd, c, d)
    out = _a(gc, gd, c, d)
    assert abs(out[0] - psnr) <= PSNR_REL * abs(psnr)
    assert abs(out[1] - ssim) <= SSIM_ABS
    assert abs(out[2] - dl1) <= DEPTH_REL * abs(dl1)
    return out


@pytest.mark.parametrize('case', ['synthetic', 'noisy', 'random_odd', 'random_min',
                                  'random_odd_nodepth', 'random_wide'])
def test_kernel_order_against_reference_semantics(case):
    rng = np.random.default_rng(7)
    if case == 'synthetic':
        gc, gd, c, d = _synthetic(480, 640)
    elif case == 'noisy':
        gc, gd, _, _ = _synthetic(480, 640, 1)
        c = np.clip(gc + rng.normal(0, 0.05, gc.shape), -0.1, 1.1).astype(f32)
        d = gd + rng.normal(0, 0.01, gd.shape)
    elif case == 'random_odd':
        gc, gd, c, d = _random(481, 641, 1)
    elif case == 'random_min':
        gc, gd, c, d = _random(161, 161, 2)
    elif case == 'random_odd_nodepth':
        gc, gd, c, _ = _random(481, 641, 3)
        d = None
    else:
        gc, gd, c, d = _random(200, 333, 4, noise=0.02)
    _check_against_b(gc, gd, c, d)


def test_identical_images_give_ms_ssim_one_and_infinite_psnr():
    gc, gd, _, _ = _synthetic(240, 320)
    out = _a(gc, gd, gc.copy(), gd.astype(np.float64))
    assert out[1] == 1.0 and out[0] == np.inf and out[2] == 0.0 and out[3] == 0.0
    psnr, ssim, _ = oe.save_render_imgs(gc, gd, gc.copy(), gd.astype(np.float64))
    assert psnr == np.inf and abs(ssim - 1.0) < 1e-6


def test_constant_offset_gives_analytic_psnr():
    rng = np.random.default_rng(0)
    H, W, c = 200, 240, 0.125
    g = (rng.integers(256, 768, size=(H, W, 3)) / 1024.0).astype(f32)   # exact in fp32
    out = _a(g, np.ones((H, W), f32), g + f32(c), np.ones((H, W)))
    assert out[3] == c * c
    assert abs(out[0] - (-10 * np.log10(c * c))) <= 1e-12 * abs(out[0])


def test_window_sums_to_one_and_matches_the_reference_window():
    w = oe.window()
    assert w.dtype == f32 and np.array_equal(w, w[::-1]) and w.argmax() == 5
    assert abs(float(w.astype(np.float64).sum()) - 1.0) < 1e-6
    ref = oe._fspecial_gauss_1d(11, 1.5).reshape(-1).numpy()
    assert np.abs(w.view(np.int32) - ref.view(np.int32)).max() <= 1   # at most 1 ulp apart


def test_transposed_inputs_give_the_same_ms_ssim():
    """The metric is symmetric in the axes; only fp32 summation orders change."""
    gc, gd, c, d = _random(300, 257, 5)
    a = _a(gc, gd, c, d)
    t = _a(gc.transpose(1, 0, 2).copy(), gd.T.copy(), c.transpose(1, 0, 2).copy(), d.T.copy())
    assert abs(a[1] - t[1]) <= 2e-6
    assert abs(a[0] - t[0]) <= 1e-13 * abs(a[0]) and abs(a[2] - t[2]) <= 1e-13 * abs(a[2])


def test_odd_sizes_pool_with_zero_padding():
    """avg_pool2d(2, 2, padding s % 2, count_include_pad): an odd side gains a zero border row
    or column at the start, averaged in."""
    x = np.arange(2 * 3 * 5 * 7, dtype=f32).reshape(2, 3, 5, 7)
    p = oe.pool(x)
    ref = torch.nn.functional.avg_pool2d(torch.from_numpy(x), 2, padding=[1, 1]).numpy()
    assert p.shape == (2, 3, 3, 4) and np.allclose(p, ref, rtol=1e-6, atol=0)
    assert p[0, 0, 0, 0] == x[0, 0, 0, 0] / 4
    gc, gd, c, d = _random(481, 641, 6)
    _check_against_b(gc, gd, c, d)


def test_minimum_side_is_checked():
    from xrdslam_b200 import _cabi
    from xrdslam_b200.eval_image import image_metrics
    lib = _cabi.lib()
    assert lib.xrd_eval_image_workspace_bytes(1, 160, 400) == 0
    assert lib.xrd_eval_image_workspace_bytes(1, 400, 160) == 0
    assert lib.xrd_eval_image_workspace_bytes(1, 161, 161) > 0
    st = lib.xrd_eval_image_metrics(None, None, None, None, 1, 160, 400, 0, None, None, None, 0,
                                    None)
    assert st == -1   # XRD_E_SHAPE before any pointer is looked at
    with pytest.raises(ValueError, match='160'):
        image_metrics(torch.zeros(1, 160, 400, 3), torch.zeros(1, 160, 400),
                      torch.zeros(1, 160, 400, 3), torch.zeros(1, 160, 400, dtype=torch.float64))
    gc, gd, c, d = _random(160, 200, 0)
    with pytest.raises(AssertionError):
        oe.save_render_imgs(gc, gd, c, d)


def test_depth_l1_without_valid_pixel_is_nan():
    gc, gd, c, d = _random(170, 180, 8)
    gd = np.zeros_like(gd)
    assert np.isnan(_a(gc, gd, c, d)[2])
    assert np.isnan(oe.save_render_imgs(gc, gd, c, d)[2])


def test_colours_are_masked_without_rendered_depth():
    gc, gd, c, _ = _random(190, 210, 9)
    out = _check_against_b(gc, gd, c, None)
    assert out[2] == 0.0
    c2 = c.copy()
    c2[gd == 0] = 0.7     # hidden by the mask
    assert np.array_equal(_a(gc, gd, c2, None), out)
    assert not np.array_equal(_a(gc, gd, c2, np.zeros(gd.shape)), _a(gc, gd, c, np.zeros(gd.shape)))


def test_values_outside_unit_range_are_clipped():
    gc, gd, c, d = _random(180, 200, 10, noise=0.5)
    assert c.min() < 0 and c.max() > 1
    out = _a(gc * 1.5 - 0.2, gd, c, d)
    assert np.array_equal(out, _a(np.clip(gc * 1.5 - 0.2, 0, 1), gd, np.clip(c, 0, 1), d))
    psnr, ssim, _ = oe.save_render_imgs(gc * 1.5 - 0.2, gd, c, d)
    assert abs(out[0] - psnr) <= PSNR_REL * abs(psnr) and abs(out[1] - ssim) <= SSIM_ABS


def test_no_rendered_colour_gives_none(tmp_path):
    from xrdslam_b200.common import save_render_imgs
    from xrdslam_b200.eval_image import render_metrics
    gc, gd, _, d = _random(170, 170, 11)
    assert render_metrics(gc, gd, None, d) is None
    assert save_render_imgs(0, gc, gd, None, d, str(tmp_path)) is None
    assert oe.save_render_imgs(gc, gd, None, d) is None
