import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA (H100) device')
    config.addinivalue_line(
        'markers', 'needs_reference: needs /root/reference (build container)')


def pytest_collection_modifyitems(config, items):
    from oracle import ref_harness
    have_ref = ref_harness.available()
    skip_ref = pytest.mark.skip(reason='/root/reference not present')
    for item in items:
        if 'needs_reference' in item.keywords and not have_ref:
            item.add_marker(skip_ref)


@pytest.fixture(scope='session')
def cuda_dev():
    import torch
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from xrdslam_b200 import _cabi
    _cabi.check('xrd_check_device', _cabi.lib().xrd_check_device(0))
    return torch.device('cuda:0')
