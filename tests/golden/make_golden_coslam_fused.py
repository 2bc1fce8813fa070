"""Record tests/golden/coslam_fused_digests.json: digests of the deterministic outputs of the
Co-SLAM fused kernels on the cases tests/test_coslam_fused_digest_gpu.py runs.

Needs a CUDA device.  Run it on the commit whose bits the kernels are pinned to.

    python tests/golden/make_golden_coslam_fused.py [OUT.json]
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

import torch  # noqa: E402

import test_coslam_fused_digest_gpu as T  # noqa: E402


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else T.DIGESTS
    dev = torch.device('cuda:0')
    store = {T.case_key(*c): T.fused_digests(dev, *c) for c in T.all_cases()}
    os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
    with open(out, 'w') as f:
        json.dump(store, f, indent=1, sort_keys=True)
        f.write('\n')
    print('wrote', out, len(store), 'cases')


if __name__ == '__main__':
    main()
