"""Record tests/golden/vox_grid_digests.json: digests of what the reference's OWN `grid` CUDA
extension (svo_intersect, inverse_cdf_sampling) returns on the inputs that
tests/test_voxfusion_gpu.py builds.

Needs a CUDA device and the extension compiled from the reference sources by
oracle/build_ref.py (oracle/_ref/grid.so).  Each grid-backed test runs once with the real
extension behind it; the test's own assertions compare the package's kernels against the
extension's outputs while they are being recorded.

    python tests/golden/make_golden_vox_grid.py [OUT.json]
"""
import importlib.machinery
import importlib.util
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

import torch  # noqa: E402

import test_voxfusion_gpu as T  # noqa: E402


def load_grid():
    path = os.path.join(ROOT, 'oracle', '_ref', 'grid.so')
    loader = importlib.machinery.ExtensionFileLoader('grid', path)
    spec = importlib.util.spec_from_loader('grid', loader)
    mod = importlib.util.module_from_spec(spec)
    loader.exec_module(mod)
    return mod


class Recorder:
    def __init__(self, key, impl, store):
        self.calls = store.setdefault(key, [])
        self.impl = impl

    def _call(self, name, *args):
        outs = getattr(self.impl, name)(*args)
        torch.cuda.synchronize()
        d_in, d_out = T.call_digests(name, args, outs)
        self.calls.append({'fn': name, 'inputs': d_in, 'outputs': d_out})
        return outs

    def svo_intersect(self, *args):
        return self._call('svo_intersect', *args)

    def inverse_cdf_sampling(self, *args):
        return self._call('inverse_cdf_sampling', *args)


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else T.DIGESTS
    grid = load_grid()
    store = {}
    T.ref_grid = lambda key, model: Recorder(key, grid, store)
    dev = torch.device('cuda:0')
    T.test_intersect_kernel_bit_exact_vs_reference_grid(dev)
    T.test_sampling_kernel_bit_exact_vs_reference_grid(dev)
    for R in (300, 5 * 1024):
        T.test_full_step_vs_oracle_chained_through_reference_grid(dev, R)
    os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
    with open(out, 'w') as f:
        json.dump(store, f, indent=1, sort_keys=True)
        f.write('\n')
    print('wrote', out, {k: len(v) for k, v in store.items()})


if __name__ == '__main__':
    main()
