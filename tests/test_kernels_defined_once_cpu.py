"""Every kernel of the library is compiled into exactly one of its cubins: one copy of its code,
one set of launch attributes.  CUB's kernels are the exception: each source that calls a CUB
algorithm instantiates its own copy of the templates.  Reads the built library only; no GPU
needed."""
import collections
import os
import re
import shutil
import subprocess

import pytest


def test_each_kernel_is_compiled_once():
    from xrdslam_b200.build import LIB_PATH
    exe = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(exe):
        pytest.skip('cuobjdump not available')
    assert os.path.exists(LIB_PATH), 'build the library first (python -m xrdslam_b200.build)'
    out = subprocess.run([exe, '-res-usage', LIB_PATH], capture_output=True, text=True,
                         check=True).stdout
    names = [n for n in re.findall(r'Function (\S+?):', out) if not n.startswith('_ZN3cub')]
    assert any(n.startswith('_ZN3xrd') for n in names), names
    copies = {n: c for n, c in collections.Counter(names).items() if c > 1}
    assert not copies, copies
