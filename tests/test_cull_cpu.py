"""cull_mesh's restatements (oracle/cull.py) on the CPU: (b) against the reference's own
cull_mesh bit for bit, (a) against (b) under the borderline rule, analytic visibility cases and
the compaction semantics."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import cull as oc

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))
import make_golden_cull as mg  # noqa: E402

f32 = np.float32
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'cull_mesh_ref.npz')


def _golden():
    return dict(np.load(GOLDEN))


def _case_args(g, use_est):
    ds = mg.Dataset(g['depth'], g['poses'], g['camera'])
    est = [torch.from_numpy(p) for p in g['est']] if use_est else None
    poses = g['est'] if use_est else g['poses']
    return ds, est, poses


def _w2c(poses):
    return np.stack([torch.inverse(torch.from_numpy(np.asarray(p, f32)))[:3].numpy() for p in poses])


def borderline_check(seen, seen_ref, verts, w2c, depth, cam, trunc, eval_rec):
    """The borderline rule: every disagreement is a borderline vertex, and they are < 0.1 % of V.
    -> the number of disagreements."""
    dis = np.nonzero(np.asarray(seen) != np.asarray(seen_ref))[0]
    if dis.size:
        bl = oc.borderline(verts[dis], w2c, depth, cam, trunc, eval_rec)
        assert bl.all(), f'{int((~bl).sum())} non-borderline disagreements, e.g. vertex {dis[~bl][:5]}'
    assert dis.size < 1e-3 * len(seen), (dis.size, len(seen))
    return int(dis.size)


@pytest.mark.needs_reference
@pytest.mark.parametrize('name,use_est,eval_rec,trunc', mg.CASES)
def test_torch_restatement_is_the_reference_bit_for_bit(name, use_est, eval_rec, trunc):
    g = _golden()
    seen_ref, kept_ref = mg.reference_decisions(g, use_est, eval_rec, trunc)
    assert np.array_equal(seen_ref, g[name + '_seen'])          # the fixture is current
    assert np.array_equal(kept_ref, g[name + '_kept'])
    ds, est, _ = _case_args(g, use_est)
    seen = oc.reference_seen(ds, g['verts'], est, eval_rec, trunc).numpy()
    assert np.array_equal(seen, seen_ref)
    assert np.array_equal(seen[g['faces']].any(1), kept_ref)


@pytest.mark.parametrize('name,use_est,eval_rec,trunc', mg.CASES)
def test_numpy_restatement_agrees_with_torch_and_the_golden(name, use_est, eval_rec, trunc):
    g = _golden()
    ds, est, poses = _case_args(g, use_est)
    w2c = _w2c(poses)
    n = len(poses)
    seen_a = oc.visible(g['verts'], w2c, g['depth'][:n], ds.cam, trunc, eval_rec)
    seen_b = oc.reference_seen(ds, g['verts'], est, eval_rec, trunc).numpy()
    for ref in (seen_b, g[name + '_seen']):
        nb = borderline_check(seen_a, ref, g['verts'], w2c, g['depth'][:n], ds.cam, trunc, eval_rec)
        print(f'{name}: {nb} borderline disagreements of {seen_a.size}')
    assert 0 < seen_a.sum() < seen_a.size


# ---- analytic cases: one frame, camera at the origin looking down -z (c2w = I) -----------------
class _Cam:
    def __init__(self, W=16, H=12, fx=10.0, fy=10.0, cx=8.0, cy=6.0):
        self.width, self.height, self.fx, self.fy, self.cx, self.cy = W, H, fx, fy, cx, cy


def _one_frame(verts, cam, depth, eval_rec=True, trunc=0.06):
    w2c = np.eye(4, dtype=f32)[None, :3]
    d = np.asarray(depth, f32)[None]
    seen_a = oc.visible(np.asarray(verts, f32), w2c, d, cam, trunc, eval_rec)
    ds = mg.Dataset(d, np.eye(4, dtype=f32)[None], [cam.height, cam.width, cam.fx, cam.fy,
                                                    cam.cx, cam.cy])
    seen_b = oc.reference_seen(ds, np.asarray(verts, f32), None, eval_rec, trunc).numpy()
    assert np.array_equal(seen_a, seen_b)
    return seen_a


def _z_cam(z):
    """A camera z whose z + f32(1e-5) is exactly `z` in float32."""
    zc = f32(z) - f32(1e-5)
    while zc + f32(1e-5) != f32(z):
        zc = np.nextafter(zc, f32(z) if zc + f32(1e-5) < f32(z) else f32(-np.inf), dtype=f32)
    return zc


def analytic_cases():
    """(name, vertices, camera, depth, eval_rec, truncation, expected seen) -- shared with the
    GPU test."""
    cam = _Cam()
    flat = np.full((cam.height, cam.width), 1.0, f32)
    cases = []
    # behind the camera, and camera -z in [0, 1e-5) (z = zc + 1e-5 > 0): not seen; -z = 1e-5
    # (x, y offset so that u, v land near the centre despite the tiny z): seen
    ox, oy = -8e-6, 6e-6
    cases.append(('behind_and_near_plane',
                  [[0, 0, 1.0], [ox, oy, -0.5e-5], [ox, oy, 0.0], [ox, oy, -2e-5], [0, 0, -0.5]],
                  cam, flat, True, 0.06, [False, False, False, True, True]))
    # u = 0 and u = W exactly (x = 0, cx = 0 or W; z a power of two): outside; just inside: seen
    for cx, expect in ((0.0, False), (16.0, False), (15.5, True), (0.5, True)):
        c = _Cam(cx=cx)
        cases.append((f'u_edge_cx{cx}', [[0, 0, _z_cam(-2.0)]], c, np.full((12, 16), 2.0, f32),
                      True, 0.06, [expect]))
    for cy, expect in ((0.0, False), (12.0, False), (11.5, True)):
        c = _Cam(cy=cy)
        cases.append((f'v_edge_cy{cy}', [[0, 0, _z_cam(-2.0)]], c, np.full((12, 16), 2.0, f32),
                      True, 0.06, [expect]))
    # occluded by less / more than the truncation behind depth 1.0
    cases.append(('occlusion', [[0, 0, -1.05], [0, 0, -1.07], [0, 0, -0.5]], cam, flat, True,
                  0.06, [True, False, True]))
    cases.append(('occlusion_t0.1', [[0, 0, -1.05], [0, 0, -1.07], [0, 0, -1.2]], cam, flat,
                  True, 0.1, [True, True, False]))
    # eval_rec off: the depth term is dropped
    cases.append(('no_eval_rec', [[0, 0, -1.05], [0, 0, -1.07], [0, 0, -50.0], [0, 0, 1.0]], cam,
                  flat, False, 0.06, [True, True, True, False]))
    # over a block of depth-0 pixels: bilinear blend is 0, so only vertices within the truncation
    # of the camera are seen
    hole = flat.copy()
    hole[3:9, 5:11] = 0.0
    cases.append(('invalid_depth', [[0, 0, -0.05], [0, 0, -0.07], [0, 0, -1.0]], cam, hole, True,
                  0.06, [True, False, False]))
    cases.append(('invalid_depth_edge', [[0, 0, -0.55], [0, 0, -0.57]], cam, _edge_depth(cam),
                  True, 0.06, [True, False]))
    return cases


def _edge_depth(cam):
    """Depth 1 in columns 0..7, 0 (invalid) from column 8 on.  The vertex (0, 0, z) projects to
    u = cx = 8, sampled at 8 * 15 / 16 = 7.5 (exact in f32): half on the last valid column, half
    on the first invalid one, so d = 0.5.  Reading pixel u (d = 0) or the nearest valid pixel
    (d = 1) would decide -z = 0.55 or 0.57 differently."""
    d = np.zeros((cam.height, cam.width), f32)
    d[:, :8] = 1.0
    return d


def test_invalid_pixels_take_part_in_the_blend():
    cam = _Cam()
    d = oc._sample_depth(_edge_depth(cam), np.array([8.0], f32), np.array([6.0], f32), 12, 16)
    assert d.tolist() == [0.5]


@pytest.mark.parametrize('case', analytic_cases(), ids=lambda c: c[0])
def test_analytic_visibility(case):
    _, verts, cam, depth, eval_rec, trunc, expect = case
    assert _one_frame(verts, cam, depth, eval_rec, trunc).tolist() == expect


def test_depth_sample_quirk_reads_u_times_w_minus_1_over_w():
    # a depth ramp along u: the sample at u is the ramp at u * (W - 1) / W, not at u
    cam = _Cam(W=16, H=12, cx=8.0)
    ramp = np.tile(np.arange(16, dtype=f32), (12, 1))
    u = np.array([3.0, 8.0, 12.5], f32)
    d = oc._sample_depth(ramp, u, np.full(3, 6.0, f32), 12, 16)
    np.testing.assert_allclose(d, u * 15 / 16, rtol=1e-6)


# ---- compaction -------------------------------------------------------------------------------
def test_compaction_semantics():
    verts = np.arange(24, dtype=f32).reshape(8, 3)
    colors = (np.arange(24) * 7 % 256).astype(np.uint8).reshape(8, 3)
    faces = np.array([[0, 1, 2], [3, 4, 5], [1, 6, 2], [5, 0, 3]], np.int32)
    seen = np.array([0, 0, 1, 0, 0, 0, 1, 1], bool)   # 7 is seen but in no face; 5 is unseen
    v, f, c = oc.compact(seen, verts, faces, colors)
    # faces 0 and 2 keep (vertex 2 / 6 seen), 1 and 3 go; 0, 1, 2, 6 are referenced, in order
    assert np.array_equal(v, verts[[0, 1, 2, 6]])
    assert np.array_equal(c, colors[[0, 1, 2, 6]])
    assert np.array_equal(f, [[0, 1, 2], [1, 3, 2]])
    assert f.dtype == np.int32
    v, f, c = oc.compact(np.zeros(8, bool), verts, faces, colors)
    assert v.shape == (0, 3) and f.shape == (0, 3) and c.shape == (0, 3)
    v, f, c = oc.compact(np.ones(8, bool), verts, faces[:, :], None)
    assert np.array_equal(v, verts[:7]) and np.array_equal(f, faces) and c is None
