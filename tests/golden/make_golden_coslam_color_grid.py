"""Record tests/golden/coslam_color_grid_step.npz: what the reference's own JointEncoding with a
separate colour grid (oneGrid=False) returns on the inputs of test_coslam_color_grid_cpu.py's
color_grid_case(): outputs, the four loss terms and the gradients of both hash tables, the four
decoder weights and the rays.  The parameters are rebuilt from seeds by the tests; the table
gradients are stored sparsely (the entries a 16-ray batch touches).

Needs the reference checkout (oracle/ref_harness.py); runs on the CPU.

    python tests/golden/make_golden_coslam_color_grid.py [OUT.npz]
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

import numpy as np  # noqa: E402

import test_coslam_color_grid_cpu as TC  # noqa: E402


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, 'coslam_color_grid_step.npz')
    rec = TC.run_reference_step()
    np.savez_compressed(out, **rec)
    print('wrote', out, {k: v.shape for k, v in rec.items()})


if __name__ == '__main__':
    main()
