"""Co-SLAM grouped fused kernel (k_fused_g, compact OneBlob record) against the tile kernel
(k_fused) on the same seeded batches, plus the compiled form of both kernels: no instantiation
copies the ~730-byte kernel-parameter block to local memory."""
import os
import re
import shutil
import subprocess

import pytest
import torch

from helpers import coslam_pair, make_rays, max_abs, rel_err

pytestmark = pytest.mark.gpu

# DESIGN.md section 2, precision mode 0 (3xTF32 everywhere)
TOL_OUT = 2e-5     # abs
TOL_LOSS = 2e-5    # rel
TOL_GRAD = 2e-4    # rel l2


def _cuobjdump():
    exe = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(exe):
        pytest.skip('cuobjdump not available')
    return exe


def test_fused_kernels_keep_parameters_out_of_local_memory():
    from xrdslam_b200.build import LIB_PATH
    exe = _cuobjdump()
    res = subprocess.run([exe, '-res-usage', LIB_PATH], capture_output=True, text=True).stdout
    lines = res.splitlines()
    found = {}
    for i, line in enumerate(lines):
        m = re.search(r'Function (_ZN3xrd6coslam(?:7k_fused|9k_fused_g)I\S*?):', line)
        if m:
            usage = line + ' ' + (lines[i + 1] if i + 1 < len(lines) else '')
            st = re.search(r'STACK:(\d+)', usage)
            assert st is not None, usage
            found[m.group(1)] = int(st.group(1))
    assert sum('k_fused_g' in k for k in found) == 5, sorted(found)
    assert sum('7k_fused' in k for k in found) == 5, sorted(found)
    # a by-reference Params argument of the non-inlined hash backward used to cost a 776..984 B
    # stack frame; what is left are register spills of the grouped backward (< 256 B)
    assert all(v < 256 for v in found.values()), found
    tile_bwd = [k for k in found if '7k_fusedILb1' in k]
    assert tile_bwd and all(found[k] == 0 for k in tile_bwd), found


def _run(model, R, seed, with_grads):
    rays_o, rays_d, ts, td, noise = make_rays(R, seed=seed)
    dev = model.embed_fn.params.device
    w = model._weights()
    return model._launch(rays_o.to(dev), rays_d.to(dev), model.embed_fn.params, *w,
                         ts.to(dev), td.to(dev), noise.to(dev), with_grads=with_grads)


def _pair(cuda_dev):
    _, tile = coslam_pair(cuda_dev, rays_per_tile=-1)
    _, grouped = coslam_pair(cuda_dev, rays_per_tile=-2)
    return tile, grouped


# 4096: the benchmark batch (2-ray units); 4097: the last unit holds one ray and is taken by a
# group whose rows are dirty from a 2-ray unit; 793: one unit more than 3 groups x 132 SMs
@pytest.mark.parametrize('R', [4096, 4097, 793])
def test_grouped_matches_tile_kernel_with_grads(cuda_dev, R):
    tile, grouped = _pair(cuda_dev)
    o_t, g_t = _run(tile, R, R, True)
    o_g, g_g = _run(grouped, R, R, True)
    torch.cuda.synchronize()
    assert torch.equal(o_g['z_vals'], o_t['z_vals'])
    for k in ('rgb', 'depth', 'acc_map', 'depth_var', 'raw'):
        assert max_abs(o_g[k], o_t[k]) < TOL_OUT, k
    for a, b in zip(o_g['losses'].tolist(), o_t['losses'].tolist()):
        assert abs(a - b) <= TOL_LOSS * max(abs(b), 1e-6), (a, b)
    for k in ('d_table', 'd_w_sdf0', 'd_w_sdf1', 'd_w_col0', 'd_w_col1', 'd_rays_o', 'd_rays_d'):
        assert rel_err(g_g[k], g_t[k]) < TOL_GRAD, k


@pytest.mark.parametrize('R', [4096, 4097])
def test_grouped_forward_bit_identical_to_tile_kernel(cuda_dev, R):
    tile, grouped = _pair(cuda_dev)
    o_t, _ = _run(tile, R, R + 1, False)
    o_g, _ = _run(grouped, R, R + 1, False)
    torch.cuda.synchronize()
    for k in ('rgb', 'depth', 'raw'):
        assert torch.equal(o_g[k], o_t[k]), k


def test_compact_oneblob_outside_the_box(cuda_dev):
    """Sample points far outside the bounding box (normalised coordinates < 0 and > 1) take the
    compact OneBlob through every branch; the forward stays bit-identical to the dense form."""
    tile, grouped = _pair(cuda_dev)
    R = 512
    rays_o, rays_d, ts, td, noise = make_rays(R, seed=7)
    rays_o = rays_o * 12.0  # most rays start outside BOUND
    dev = cuda_dev
    outs = []
    for m in (tile, grouped):
        w = m._weights()
        o, _ = m._launch(rays_o.to(dev), rays_d.to(dev), m.embed_fn.params, *w, ts.to(dev),
                         td.to(dev), noise.to(dev), with_grads=False)
        outs.append(o)
    torch.cuda.synchronize()
    for k in ('rgb', 'depth', 'raw'):
        assert torch.equal(outs[1][k], outs[0][k]), k
