"""Compiled form of the Co-SLAM fused kernels.  The grouped kernel's (k_fused_g) gradient
instantiations keep the weight-gradient accumulators out of local memory and stay in the 196 KB
shared-memory configuration of an sm_90 SM; the tile kernel's (k_fused) keep a 0-byte stack frame.
Reads the built library only; no GPU needed."""
import os
import re
import shutil
import subprocess

import pytest

# dynamic shared memory of a gradient pass with map gradients (G_SMEM_DW in csrc/coslam.cu)
SMEM_DYNAMIC = 198_784
CARVEOUT_196K = 196 * 1024


def _res_usage(kernel=r'9k_fused_gILb1'):
    """{mangled name: {REG, STACK, SHARED}} of the gradient instantiations (precision modes 0, 1,
    2) of the kernel whose mangled name continues _ZN3xrd6coslam with `kernel`."""
    from xrdslam_b200.build import LIB_PATH
    exe = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(exe):
        pytest.skip('cuobjdump not available')
    assert os.path.exists(LIB_PATH), 'build the library first (python -m xrdslam_b200.build)'
    lines = subprocess.run([exe, '-res-usage', LIB_PATH], capture_output=True, text=True,
                           check=True).stdout.splitlines()
    found = {}
    for i, line in enumerate(lines):
        m = re.search(r'Function (_ZN3xrd6coslam' + kernel + r'\S*?):', line)
        if m:
            usage = lines[i + 1] if i + 1 < len(lines) else ''
            found[m.group(1)] = {k: int(v) for k, v in re.findall(r'(REG|STACK|SHARED):(\d+)', usage)}
    assert len(found) == 3, sorted(found)  # precision modes 0, 1, 2
    return found


def test_grouped_gradient_kernels_do_not_spill():
    # with all 28 weight-gradient accumulators in registers these had a 120 B stack frame
    for name, u in _res_usage().items():
        assert u['STACK'] <= 16, (name, u)
        assert u['REG'] <= 96, (name, u)  # 576 threads per SM


def test_grouped_gradient_kernels_fit_the_196k_carveout():
    # SHARED: static shared memory plus the per-CTA reservation
    for name, u in _res_usage().items():
        assert SMEM_DYNAMIC + u['SHARED'] <= CARVEOUT_196K, (name, u)


def test_tile_gradient_kernels_do_not_spill():
    # at ~240 registers a spill would put local-memory traffic into the per-ray composite and the
    # weight-gradient loops
    for name, u in _res_usage(r'7k_fusedILb1').items():
        assert u['STACK'] == 0, (name, u)
