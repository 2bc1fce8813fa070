"""oracle/ingest.py (the restatement csrc/ingest.cu is tested against) against the reference's
frame transform run with real cv2 (tests/golden/ingest_ref.npz, make_golden_ingest.py)."""
import json
import os

import numpy as np
import pytest

from oracle import ingest as O

GOLDEN = os.path.join(os.path.dirname(__file__), 'golden', 'ingest_ref.npz')
# Cases whose colour goes through a non-trivial INTER_LINEAR resize of float64 data.  There cv2's
# default build hands the resize to Intel IPP, whose arithmetic is not cv2's own C++ code; the
# oracle follows cv2's own code, which cv2 runs with IPP switched off (`*_noipp`, the same bits
# as with optimisations off), and reproduces it bit for bit.  Against the IPP resize the
# largest difference measured on the recorded cases is 1.55e-6 (combined), about 26 float32 ulp at
# the value's magnitude; every other case and every depth map is bit-identical to all three.
IPP_RESIZE_CASES = {'colour_larger', 'down2_odd', 'down3_odd', 'combined'}
IPP_RESIZE_MAX_ABS = 2e-6


def _bits_equal(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return a.shape == b.shape and np.array_equal(a.view(np.int32), b.view(np.int32))


def _cases():
    g = np.load(GOLDEN)
    return g, json.loads(str(g['meta']))['cases']


def _oracle(g, name):
    fx, fy, cx, cy, s, e, f = g[name + '/camera']
    dist = g[name + '/dist']
    return O.ingest(g[name + '/color'], g[name + '/depth_u16'], fx, fy, cx, cy,
                    dist if dist.size else None, s, int(e), int(f))


def test_golden_fixture_is_small():
    assert os.path.getsize(GOLDEN) < 1 << 20


def test_oracle_matches_cv2_without_ipp_bit_exact():
    g, cases = _cases()
    assert len(cases) == 8
    for name in cases:
        rgb, dep = _oracle(g, name)
        assert _bits_equal(rgb, g[name + '/rgb_noipp']), name
        assert _bits_equal(dep, g[name + '/depth_noipp']), name


def test_oracle_against_cv2_with_ipp():
    g, cases = _cases()
    for name in cases:
        rgb, dep = _oracle(g, name)
        ref = g[name + '/rgb']
        assert _bits_equal(dep, g[name + '/depth']), name
        if name in IPP_RESIZE_CASES:
            assert rgb.shape == ref.shape
            assert np.abs(rgb - ref).max() <= IPP_RESIZE_MAX_ABS, name
        else:
            assert _bits_equal(rgb, ref), name


def test_output_sizes():
    g, cases = _cases()
    for name in cases:
        _, _, _, _, _, e, f = g[name + '/camera']
        h, w = O.output_size(*g[name + '/depth_u16'].shape, int(e), int(f))
        assert g[name + '/rgb'].shape == (h, w, 3) and g[name + '/depth'].shape == (h, w)


def test_distortion_coefficient_counts():
    for n in (4, 5, 8, 12):
        assert O.dist_coeffs(np.arange(n) * 0.01)[:n].tolist() == (np.arange(n) * 0.01).tolist()
    with pytest.raises(ValueError):
        O.dist_coeffs([0.1] * 6)


def test_oracle_matches_live_cv2_generic():
    """Seeded random shapes, intrinsics, distortion, crops and factors against cv2 itself (its own
    C++ code: optimisations, and with them IPP, off), when cv2 is installed."""
    cv2 = pytest.importorskip('cv2')
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(__file__), 'golden'))
    from make_golden_ingest import reference_transform
    rng = np.random.default_rng(5)
    opt = cv2.useOptimized()
    cv2.setUseOptimized(False)
    try:
        for _ in range(40):
            Hd, Wd = (int(v) for v in rng.integers(20, 90, 2))
            H0, W0 = ((Hd, Wd) if rng.random() < 0.5 else
                      tuple(int(v) for v in rng.integers(20, 140, 2)))
            color = rng.integers(0, 256, (H0, W0, 3), dtype=np.uint8)
            depth = rng.integers(0, 65536, (Hd, Wd), dtype=np.uint16)
            fx, fy = (float(v) for v in rng.uniform(0.5, 1.5, 2) * W0)
            cx, cy = float(rng.uniform(0.3, 0.7) * W0), float(rng.uniform(0.3, 0.7) * H0)
            dist = (list(rng.normal(0, 0.1, int(rng.choice([4, 5, 8, 12]))))
                    if rng.random() < 0.5 else None)
            e, f = int(rng.integers(0, 4)), int(rng.choice([1, 2, 3]))
            args = (fx, fy, cx, cy, 1000.0, e, f, dist)
            rgb, dep = reference_transform(color.copy(), depth.copy(), *args)
            orgb, odep = O.ingest(color, depth, fx, fy, cx, cy, dist, 1000.0, e, f)
            assert _bits_equal(orgb, rgb) and _bits_equal(odep, dep)
    finally:
        cv2.setUseOptimized(opt)
