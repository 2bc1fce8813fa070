"""Record tests/golden/coslam_importance_step.npz: what the reference's own JointEncoding with
importance sampling (training_n_importance > 0) returns on the inputs of
test_coslam_importance_cpu.py's importance_case(), for its GOLDEN_CASES (N = 5 with the det
draw, training_perturb = 0; N = 16 with the random draw): outputs, the coarse outputs, z_std,
the four loss terms and the gradients of the hash table, the four decoder weights and the rays,
under the prefix 'n{N}_det{0|1}/'.  The parameters are rebuilt from seeds by the tests; the
table gradients are stored sparsely.

Needs the reference checkout (oracle/ref_harness.py); runs on the CPU.

    python tests/golden/make_golden_coslam_importance.py [OUT.npz]
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

import numpy as np  # noqa: E402

import test_coslam_importance_cpu as TI  # noqa: E402


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, 'coslam_importance_step.npz')
    rec = {}
    for N, det in TI.GOLDEN_CASES:
        rec.update({f'n{N}_det{int(det)}/{k}': v for k, v in TI.run_reference_step(N, det).items()})
    np.savez_compressed(out, **rec)
    print('wrote', out, os.path.getsize(out), 'bytes')


if __name__ == '__main__':
    main()
