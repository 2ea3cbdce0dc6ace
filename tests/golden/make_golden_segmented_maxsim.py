"""Writes tests/golden/segmented_maxsim.npz: what the reference's OWN segmented_maxsim.cpp returns on the seeded
scores of tests/test_oracle.py::test_segmented_maxsim_matches_reference_extension_golden.

Needs the reference extension compiled into oracle/_ref/ (python oracle/build_ref.py, which reads the reference
checkout), so it runs only where that checkout exists:

    python tests/golden/make_golden_segmented_maxsim.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))


def main():
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import build_ref
    build_ref.build_one("segmented_maxsim_cpp")
    mod = build_ref.load("segmented_maxsim_cpp")
    if mod is None:
        raise SystemExit("oracle/_ref/segmented_maxsim_cpp.so not available: the reference checkout is needed")
    # the same inputs the test regenerates from the seed
    rng = np.random.default_rng(1)
    lengths = rng.integers(1, 40, size=50)
    scores = rng.standard_normal((int(lengths.sum()), 33)).astype(np.float32)
    ref = mod.segmented_maxsim_cpp(torch.from_numpy(scores), torch.from_numpy(lengths).long()).numpy()
    out = os.path.join(HERE, "segmented_maxsim.npz")
    np.savez_compressed(out, ref=ref)
    print(out, ref.shape, ref.dtype)


if __name__ == "__main__":
    main()
