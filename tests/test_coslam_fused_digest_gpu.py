"""Co-SLAM fused kernels pinned bit for bit: SHA-256 digests of the deterministic outputs of
both fused kernels (tile -1, grouped -2), in every precision mode, at two batch sizes and for
the forward-only, pose-only and full-gradient passes.  tests/golden/make_golden_coslam_fused.py
recorded tests/golden/coslam_fused_digests.json from these same runs.

Digested: z_vals, rgb, depth, acc_map, depth_var, raw and, where the pass computes them,
d_rays_o / d_rays_d (per-ray warp sums in a fixed order).  Losses, d_table and d_w_* are left
out: they are accumulated with unordered float atomics."""
import functools
import json
import os

import pytest
import torch

from helpers import coslam_pair, digest, make_rays

pytestmark = pytest.mark.gpu

DIGESTS = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden',
                       'coslam_fused_digests.json')
KERNELS = (-1, -2)
PRECISIONS = (0, 1, 2)
RAYS = (1024, 4097)
PASSES = ('fwd', 'pose', 'full')
OUTPUTS = ('z_vals', 'rgb', 'depth', 'acc_map', 'depth_var', 'raw')
RAY_GRADS = ('d_rays_o', 'd_rays_d')


def case_key(kernel, precision, R, pass_):
    return f'{kernel}/{precision}/{R}/{pass_}'


@functools.lru_cache(maxsize=None)
def _model(dev):
    return coslam_pair(dev, seed=1)[1]


def fused_digests(dev, kernel, precision, R, pass_):
    """{output name: digest} of one fused step on coslam_pair(seed=1) and make_rays(R, seed=R)."""
    model = _model(dev)
    model.config.rays_per_tile = kernel
    model.config.precision = precision
    rays_o, rays_d, ts, td, noise = make_rays(R, seed=R)
    o, g = model._launch(rays_o.to(dev), rays_d.to(dev), model.embed_fn.params,
                         *model._weights(), ts.to(dev), td.to(dev), noise.to(dev),
                         with_grads=pass_ != 'fwd', map_grads=pass_ == 'full')
    torch.cuda.synchronize()
    out = {k: digest(o[k]) for k in OUTPUTS}
    if g is not None:
        out.update({k: digest(g[k]) for k in RAY_GRADS})
    return out


def all_cases():
    return [(k, p, R, s) for k in KERNELS for p in PRECISIONS for R in RAYS for s in PASSES]


@pytest.mark.parametrize('kernel,precision,R,pass_', all_cases())
def test_fused_outputs_match_recorded_digests(cuda_dev, kernel, precision, R, pass_):
    with open(DIGESTS) as f:
        want = json.load(f)[case_key(kernel, precision, R, pass_)]
    got = fused_digests(cuda_dev, kernel, precision, R, pass_)
    assert got == want
