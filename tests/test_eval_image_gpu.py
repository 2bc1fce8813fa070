"""Render-quality metrics on the device (csrc/eval_image.cu, eval_image.py): the kernels bit for
bit against their numpy restatement (oracle/eval_image.py (a)), against the torch restatement of
the reference (b) within the gates of test_eval_image_cpu.py, status codes, save_render_imgs end
to end, render_img(to_host=False), and Algorithm.eval_re_render for the four algorithms."""
import warnings

import numpy as np
import pytest
import torch

from oracle import eval_image as oe
from test_eval_image_cpu import DEPTH_REL, PSNR_REL, SSIM_ABS, _random

pytestmark = pytest.mark.gpu
f32 = np.float32


def _batch(kind, B, H, W):
    if kind == 'synthetic':
        from xrdslam_b200.synthetic import make_sequence
        _, _, fr = make_sequence(B + 1, width=W, height=H)
        gc = np.stack([fr[k][0] for k in range(B)])
        gd = np.stack([fr[k][1] for k in range(B)])
        c = np.stack([fr[k + 1][0] for k in range(B)])
        d = np.stack([fr[k + 1][1] for k in range(B)]).astype(np.float64)
    else:
        parts = [_random(H, W, 100 * B + k) for k in range(B)]
        gc, gd, c, d = (np.stack([p[i] for p in parts]) for i in range(4))
    return gc, gd, c, d


def _device_metrics(dev, gc, gd, c, d):
    from xrdslam_b200.eval_image import image_metrics
    t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a)).to(dev, dt)
    B = gd.shape[0]
    levels = torch.empty(B, 5, 3, 2, dtype=torch.float64, device=dev)
    out = image_metrics(t(gc, torch.float32), t(gd, torch.float32), t(c, torch.float32),
                        None if d is None else t(d, torch.float64), levels=levels)
    return out.cpu().numpy(), levels.cpu().numpy()


def _same_bits(a, b):
    a, b = np.ascontiguousarray(a, np.float64), np.ascontiguousarray(b, np.float64)
    return np.array_equal(a.view(np.uint64), b.view(np.uint64))


@pytest.mark.parametrize('kind,B,H,W,depth', [
    ('synthetic', 1, 480, 640, True), ('synthetic', 8, 480, 640, True),
    ('random', 1, 480, 640, True), ('random', 8, 480, 640, False),
    ('random', 1, 481, 641, True), ('random', 8, 481, 641, True),
    ('random', 1, 161, 161, False), ('random', 8, 161, 161, True),
    ('synthetic', 8, 161, 200, True)])
def test_kernels_bit_exact_against_numpy_restatement(cuda_dev, kind, B, H, W, depth):
    gc, gd, c, d = _batch(kind, B, H, W)
    if not depth:
        d = None
    got, got_lv = _device_metrics(cuda_dev, gc, gd, c, d)
    exp, exp_lv = oe.metrics(gc, gd, c, d)
    assert _same_bits(got_lv, exp_lv)
    assert _same_bits(got[:, 2:], exp[:, 2:])         # depth_l1, mse
    # psnr = -10 log10(mse) and ms_ssim = f(pow(...)): CUDA's and numpy's log10 / pow need not
    # round alike; their inputs are bit-identical (above)
    assert np.allclose(got[:, :2], exp[:, :2], rtol=1e-14, atol=0)
    again, again_lv = _device_metrics(cuda_dev, gc, gd, c, d)
    assert _same_bits(again, got) and _same_bits(again_lv, got_lv)


@pytest.mark.parametrize('H,W', [(480, 640), (481, 641)])
def test_against_reference_semantics(cuda_dev, H, W):
    gc, gd, c, d = _batch('synthetic', 4, H, W)
    c[1] = np.clip(gc[1] + np.random.default_rng(0).normal(0, 0.05, gc[1].shape), -0.1, 1.1)
    got, _ = _device_metrics(cuda_dev, gc, gd, c, d)
    for k in range(4):
        psnr, ssim, dl1 = oe.save_render_imgs(gc[k], gd[k], c[k], d[k])
        assert abs(got[k, 0] - psnr) <= PSNR_REL * abs(psnr)
        assert abs(got[k, 1] - ssim) <= SSIM_ABS
        assert abs(got[k, 2] - dl1) <= DEPTH_REL * abs(dl1)


def test_status_codes(cuda_dev):
    from xrdslam_b200 import _cabi
    lib = _cabi.lib()
    B, H, W = 2, 170, 190
    gc, gd, c, d = (torch.from_numpy(np.ascontiguousarray(a)).to(cuda_dev)
                    for a in _batch('random', B, H, W))
    nb = lib.xrd_eval_image_workspace_bytes(B, H, W)
    assert nb > 0
    ws = torch.empty(nb, dtype=torch.uint8, device=cuda_dev)
    out = torch.full((B, 4), -7.0, dtype=torch.float64, device=cuda_dev)
    p = _cabi.ptr
    s = torch.cuda.current_stream(cuda_dev).cuda_stream

    def call(gc_=gc, d_=d, b=B, h=H, w=W, flags=0, out_=out, ws_=ws, nbytes=nb):
        return lib.xrd_eval_image_metrics(p(gc_), p(c), p(gd), p(d_), b, h, w, flags, p(out_),
                                          None, p(ws_), nbytes, s)

    assert call(b=0) == -1 and call(h=160) == -1 and call(w=160) == -1 and call(flags=2) == -1
    assert call(h=16385) == -1
    assert call(gc_=None) == -6 and call(d_=None) == -6 and call(out_=None) == -6
    assert call(ws_=None) == -6
    assert call(nbytes=nb - 1) == -3
    torch.cuda.synchronize()
    assert bool((out == -7.0).all())       # nothing was written
    assert call(d_=None, flags=1) == 0      # no rendered depth: depth may be NULL
    assert call() == 0
    torch.cuda.synchronize()
    assert bool(torch.isfinite(out).all())


def test_save_render_imgs_end_to_end(cuda_dev, tmp_path):
    from xrdslam_b200.common import save_render_imgs
    from xrdslam_b200.eval_image import render_metrics
    gc, gd, c, d = (a[0] for a in _batch('synthetic', 1, 480, 640))
    res = save_render_imgs(3, gc, gd, c, d, str(tmp_path))
    assert len(res) == 4 and all(isinstance(v, float) for v in res)
    psnr, ssim, lpips, dl1 = res
    ep, es, ed = oe.save_render_imgs(gc, gd, c, d)
    assert abs(psnr - ep) <= PSNR_REL * abs(ep) and abs(ssim - es) <= SSIM_ABS
    assert abs(dl1 - ed) <= DEPTH_REL * abs(ed) and np.isnan(lpips)
    assert list(tmp_path.iterdir()) == []           # no figure is written
    r = render_metrics(gc, gd, c, None)             # masked colours, no depth
    ep, es, ed = oe.save_render_imgs(gc, gd, c, None)
    assert abs(r['psnr'] - ep) <= PSNR_REL * abs(ep) and abs(r['ssim'] - es) <= SSIM_ABS
    assert r['depth_l1'] == 0.0
    # device tensors and a batch go through the same path
    rb = render_metrics(torch.from_numpy(gc[None]).to(cuda_dev), gd[None], c[None], d[None],
                        lpips_fn=lambda a, b: float((a - b).abs().mean()))
    assert rb['psnr'].shape == (1, ) and rb['psnr'][0] == psnr and rb['ssim'][0] == ssim
    assert abs(rb['lpips'][0] - np.abs(np.clip(gc, 0, 1) - np.clip(c, 0, 1)).mean()) < 1e-6


# ---------------------------------------------------------------- the algorithms ---
W_IMG, H_IMG, N_FRAMES = 224, 176, 5


class _Dataset:
    def __init__(self, cam, poses, frames):
        self.cam, self.poses, self.frames = cam, poses, frames

    def __len__(self):
        return len(self.frames)

    def __getitem__(self, i):
        return i, self.frames[i][0], self.frames[i][1], self.poses[i]

    def get_camera(self):
        return self.cam


def _algorithm(name, dev, width=W_IMG, height=H_IMG, n_frames=N_FRAMES):
    """A lightly mapped algorithm on the synthetic sequence and its dataset."""
    from xrdslam_b200.frame import Frame
    from xrdslam_b200.synthetic import make_sequence
    torch.manual_seed(0)
    np.random.seed(0)
    off = (10.0, 10.0, 10.0) if name == 'voxfusion' else (0.0, 0.0, 0.0)
    cam, poses, fr = make_sequence(n_frames, width=width, height=height, offset=off)
    frames = [Frame(k, fr[k][0], fr[k][1], init_pose=poses[k],
                    separate_LR=name in ('coslam', 'pointslam'),
                    rot_rep='quat' if name in ('nice', 'voxfusion') else 'axis_angle')
              for k in range(n_frames)]
    with warnings.catch_warnings():
        warnings.simplefilter('ignore', RuntimeWarning)
        warnings.simplefilter('ignore', UserWarning)
        if name == 'coslam':
            from xrdslam_b200.coslam import CoSLAMConfig
            algo = CoSLAMConfig(mapping_sample=512).setup(camera=cam, device=dev)
        elif name == 'nice':
            from xrdslam_b200.nice_slam import NiceSLAMConfig
            b = [[-3.2, 3.2], [-4.2, 2.7], [-2.2, 2.7]]
            algo = NiceSLAMConfig(mapping_bound=b, marching_cubes_bound=b,
                                  ray_batch_size=8000).setup(camera=cam, device=dev)
        elif name == 'voxfusion':
            from xrdslam_b200.voxfusion import VoxFusionConfig
            algo = VoxFusionConfig().setup(camera=cam, device=dev)
        else:
            from xrdslam_b200.point_slam import PointSLAMConfig
            algo = PointSLAMConfig(pixels_adding=1500, mapping_sample=1000).setup(camera=cam,
                                                                                  device=dev)
    if name == 'coslam':      # Co-SLAM's keyframes keep only their ray bank
        algo.optimize_update(5, [frames[0]], is_mapping=True)
        algo.add_keyframe(frames[0])
    else:
        algo.add_keyframe(frames[0])
        algo.optimize_update(5, [frames[0]], is_mapping=True)
    if name in ('pointslam', 'voxfusion'):
        # Point-SLAM: the dynamic query radius of every frame; Vox-Fusion: voxels every frame sees
        for f in frames[1:]:
            algo.pre_precessing(f, True)
    return algo, _Dataset(cam, poses, fr)


ALGOS = ['coslam', 'nice', 'voxfusion', 'pointslam']


def _rewind(algo):
    """Renders draw Philox noise from a per-call counter: two renders that must match start
    from the same counter."""
    state = getattr(algo.model, '_step_count', None)

    def reset():
        if state is not None:
            algo.model._step_count = state
    return reset


@pytest.mark.parametrize('name', ALGOS)
def test_render_img_to_host_false_gives_the_same_bits(cuda_dev, name):
    algo, ds = _algorithm(name, cuda_dev)
    reset = _rewind(algo)
    _, rgb, depth, c2w = ds[2]
    reset()
    hc, hd = algo.render_img(c2w, gt_depth=depth, idx=2)
    reset()
    dc, dd = algo.render_img(c2w, gt_depth=depth, idx=2, to_host=False)
    assert isinstance(hc, np.ndarray) and torch.is_tensor(dc) and dc.is_cuda
    assert dc.dtype == torch.float32 and dd.dtype == torch.float64
    assert np.array_equal(hc.view(np.uint32), dc.cpu().numpy().view(np.uint32))
    assert np.array_equal(hd.view(np.uint64), dd.cpu().numpy().view(np.uint64))


@pytest.mark.parametrize('name', ALGOS)
def test_eval_re_render_matches_host_loop(cuda_dev, name, capsys):
    from xrdslam_b200.eval_image import render_metrics
    algo, ds = _algorithm(name, cuda_dev)
    reset = _rewind(algo)
    calls = []

    def lpips_fn(a, b):
        calls.append(a.shape)
        return 0.25

    reset()
    res = algo.eval_re_render(ds, render_freq=2, estimate_c2w_list=ds.poses, lpips_fn=lpips_fn)
    assert [r['idx'] for r in res['frames']] == [0, 2, 4]
    assert calls == [(H_IMG, W_IMG, 3)] * 3 and res['avg_lpips'] == 0.25
    assert 'avg_psnr[dB]' in capsys.readouterr().out
    reset()
    for row in res['frames']:
        i, rgb, depth, c2w = ds[row['idx']]
        color, rdepth = algo.render_img(c2w, gt_depth=depth, idx=i)
        m = render_metrics(rgb, depth, color, rdepth)
        assert (row['psnr'], row['ssim'], row['depth_l1']) == (m['psnr'], m['ssim'],
                                                               m['depth_l1'])
        ep, es, ed = oe.save_render_imgs(rgb, depth, color, rdepth)
        assert abs(row['psnr'] - ep) <= PSNR_REL * abs(ep) and abs(row['ssim'] - es) <= SSIM_ABS
        assert abs(row['depth_l1'] - ed) <= DEPTH_REL * abs(ed)
        assert np.isfinite(row['psnr']) and 0 < row['ssim'] <= 1
    for key in ('psnr', 'ssim', 'depth_l1'):   # sequential sums, as tracker.py accumulates them
        r = res['frames']
        assert res['avg_' + key] == ((r[0][key] + r[1][key]) + r[2][key]) / 3
    res = algo.eval_re_render(ds, render_freq=4, estimate_c2w_list=ds.poses)
    assert [r['idx'] for r in res['frames']] == [0, 4]
    assert all(np.isnan(r['lpips']) for r in res['frames'])
