"""Build libxrdslam_b200.so (the C-ABI shared library) in-tree with nvcc for sm_90a (H100).

Usage: python -m xrdslam_b200.build [--force] [--verbose]
The library carries no torch dependency: plain CUDA runtime + the C-ABI in
include/xrdslam_b200.h.  Python binds it with ctypes (xrdslam_b200/_cabi.py).
"""
from __future__ import annotations

import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, 'csrc')
LIB_DIR = os.path.join(HERE, 'lib')
LIB_PATH = os.path.join(LIB_DIR, 'libxrdslam_b200.so')

NVCC_FLAGS = [
    '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-lineinfo',
    '-std=c++17', '--expt-relaxed-constexpr', '-Xcompiler', '-fPIC', '-I',
    os.path.join(ROOT, 'include'), '-I', CSRC
]


def sources():
    return sorted(
        glob.glob(os.path.join(CSRC, '*.cu')) +
        glob.glob(os.path.join(CSRC, '*.cpp')))


def _stale():
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    deps = sources() + glob.glob(os.path.join(CSRC, '*.cuh')) + glob.glob(
        os.path.join(CSRC, '*.h')) + glob.glob(
            os.path.join(ROOT, 'include', '*.h'))
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not _stale():
        return LIB_PATH
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    os.makedirs(LIB_DIR, exist_ok=True)
    objs = []
    procs = []
    for src in sources():
        obj = os.path.join(LIB_DIR,
                           os.path.basename(src).rsplit('.', 1)[0] + '.o')
        objs.append(obj)
        if (not force and os.path.exists(obj) and os.path.getmtime(obj) >
                max(os.path.getmtime(src),
                    *(os.path.getmtime(h)
                      for h in glob.glob(os.path.join(CSRC, '*.cuh')) +
                      glob.glob(os.path.join(ROOT, 'include', '*.h'))))):
            continue
        cmd = [nvcc] + NVCC_FLAGS + (['-Xptxas', '-v'] if verbose else
                                     []) + ['-x', 'cu', '-c', src, '-o', obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE,
                                            stderr=subprocess.STDOUT)))
    for src, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode != 0:
            sys.stderr.write(out.decode())
        if p.returncode != 0:
            raise RuntimeError(f'nvcc failed on {src}')
    cmd = [nvcc, '-shared', '-o', LIB_PATH] + objs + [
        '-gencode', 'arch=compute_90a,code=sm_90a', '-lcudart'
    ]
    subprocess.check_call(cmd)
    return LIB_PATH


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose='--verbose' in sys.argv))
