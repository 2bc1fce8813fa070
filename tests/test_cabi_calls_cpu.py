"""The Python side of the C-ABI has one calling protocol (xrdslam_b200/_cabi.py: call, launch,
launch_on, workspace, require_cuda).  A source scan keeps every product module on it, and a
recording stub in place of the shared library checks what the helpers hand to an entry point."""
import ast
import contextlib
import os
import re

import pytest
import torch

from xrdslam_b200 import _cabi

PKG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'xrdslam_b200')
# host-side octree calls: they return a handle, a node count or nothing, not an XrdStatus
HOST_CALLS = {'xrd_octree_create', 'xrd_octree_destroy', 'xrd_octree_num_nodes',
              'xrd_octree_insert', 'xrd_octree_export'}
WORKSPACE_SYMBOL = re.compile(r'xrd_\w*_workspace_bytes')


def _modules():
    for name in sorted(os.listdir(PKG)):
        if name.endswith('.py') and name != '_cabi.py':
            with open(os.path.join(PKG, name)) as f:
                yield name, ast.parse(f.read())


def test_product_modules_call_the_library_through_the_helpers():
    direct, sizing = [], []
    for name, tree in _modules():
        for node in ast.walk(tree):
            if isinstance(node, ast.Attribute) and node.attr.startswith('xrd_') and \
                    node.attr not in HOST_CALLS:
                direct.append(f'{name}:{node.lineno} {node.attr}')
            text = node.attr if isinstance(node, ast.Attribute) else \
                node.value if isinstance(node, ast.Constant) and isinstance(node.value, str) else \
                node.id if isinstance(node, ast.Name) else None
            if text is not None and WORKSPACE_SYMBOL.search(text):
                sizing.append(f'{name}:{node.lineno}')
    assert not direct, f'entry points called outside _cabi: {direct}'
    assert not sizing, f'workspace sizes queried outside _cabi.workspace: {sizing}'


class _StubLib:
    """Records every call with the current device at the time of the call."""

    def __init__(self, state, status=0, nbytes=0):
        self.state, self.status, self.nbytes, self.calls = state, status, nbytes, []

    def xrd_last_cuda_error(self):
        return 0

    def __getattr__(self, name):
        if not name.startswith('xrd_'):
            raise AttributeError(name)

        def fn(*args):
            self.calls.append((name, args, self.state['device']))
            return self.nbytes if name.endswith('_workspace_bytes') else self.status
        return fn


@pytest.fixture
def stub(monkeypatch):
    """_cabi with a stub library, torch.cuda.device tracking the current device and
    torch.cuda.current_stream(dev) giving a handle per device."""
    state = {'device': None}

    @contextlib.contextmanager
    def device(dev):
        prev, state['device'] = state['device'], dev
        try:
            yield
        finally:
            state['device'] = prev

    class Stream:
        def __init__(self, dev):
            self.cuda_stream = 1000 + (torch.device(dev).index or 0)

    lib = _StubLib(state)
    monkeypatch.setattr(_cabi, '_lib', lib)
    monkeypatch.setattr(torch.cuda, 'device', device)
    monkeypatch.setattr(torch.cuda, 'current_stream', Stream)
    return lib


def test_call_passes_the_arguments_and_checks_the_status(stub):
    _cabi.call('xrd_layout', 1, 2.5, None)
    assert stub.calls == [('xrd_layout', (1, 2.5, None), None)]
    stub.status = -1
    with pytest.raises(_cabi.XrdError, match='^xrd_layout failed: XRD_E_SHAPE$') as e:
        _cabi.call('xrd_layout', 1)
    assert e.value.status == -1


def test_launch_appends_the_stream_and_switches_no_device(stub):
    _cabi.launch('xrd_kernel', 7, None, stream=1234)
    assert stub.calls == [('xrd_kernel', (7, None, 1234), None)]
    stub.status = -6
    with pytest.raises(_cabi.XrdError, match='xrd_kernel failed: XRD_E_NULL'):
        _cabi.launch('xrd_kernel', 7, stream=1234)


def test_launch_on_runs_on_the_devices_current_stream_inside_its_context(stub):
    dev = torch.device('cuda:3')
    _cabi.launch_on(dev, 'xrd_kernel', 1, 2)
    assert stub.calls == [('xrd_kernel', (1, 2, 1003), dev)]
    stub.status = -3
    with pytest.raises(_cabi.XrdError, match='xrd_kernel failed: XRD_E_WORKSPACE'):
        _cabi.launch_on(dev, 'xrd_kernel', 1, 2)


def test_workspace_forwards_the_reported_size(stub):
    stub.nbytes = 4096
    ws, nb = _cabi.workspace('cpu', 'thing', 3, 4, error='never raised')
    assert nb == 4096 and ws.numel() == 4096 and ws.dtype == torch.uint8
    assert stub.calls == [('xrd_thing_workspace_bytes', (3, 4), None)]


def test_zero_workspace_is_not_null_and_error_raises(stub):
    ws, nb = _cabi.workspace('cpu', 'thing', 3)
    assert nb == 0 and ws.numel() >= 1 and ws.data_ptr() != 0
    with pytest.raises(ValueError, match='^unsupported size 3$'):
        _cabi.workspace('cpu', 'thing', 3, error='unsupported size 3')


def test_reduction_forwards_the_workspace_the_library_sized(stub):
    """A converted call site end to end: the library's byte count and a non-null buffer reach
    the entry point, on the data's device and its current stream."""
    from xrdslam_b200 import eval_recon
    d = torch.zeros(10)
    for nbytes in (512, 0):
        stub.calls.clear()
        stub.nbytes = nbytes
        eval_recon.dist_stats(d, 0.5)
        (size, size_args, _), (name, args, dev) = stub.calls
        assert (size, size_args) == ('xrd_eval_reduce_workspace_bytes', (10,))
        assert name == 'xrd_eval_dist_stats' and dev == d.device
        assert args[0] == d.data_ptr() and args[1:3] == (10, 0.5)
        assert args[4] != 0 and args[5] == nbytes and args[6] == 1000


def test_require_cuda():
    with pytest.raises(RuntimeError, match='no CPU path: values must be on a CUDA device'):
        _cabi.require_cuda(torch.device('cpu'), 'values')
    with pytest.raises(RuntimeError, match='no CPU path'):
        _cabi.require_cuda('cpu', 'values')
    _cabi.require_cuda(torch.device('cuda:1'), 'values')
    _cabi.require_cuda('cuda', 'values')
