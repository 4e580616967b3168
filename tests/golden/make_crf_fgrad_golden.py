"""Regenerate tests/golden/crf_fgrad_ref.npz: the reference CRF's own kernel_grad for a term added as
addPairwiseEnergy(features, ..., FULL_KERNEL) at P = I (built into oracle/_ref/libdensecrf_fgrad_ref.so by
oracle/fgrad.mk) on a few images, with Potts and MatrixCompatibility terms, so that the feature-gradient tests have a
pin to the reference wherever oracle/_ref was not built.  Run from the repository root:
python tests/golden/make_crf_fgrad_golden.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.join(HERE, "..", ".."), os.path.join(HERE, "..")]

from crf_fgrad_cases import GOLDEN, GOLDEN_CASES, golden_inputs  # noqa: E402
from oracle import crf_fgrad_oracle  # noqa: E402


def main():
    if not crf_fgrad_oracle.ref_available():
        sys.exit("oracle/_ref/libdensecrf_fgrad_ref.so is not built")
    out = {}
    for name in GOLDEN_CASES:
        features, unary, G, p, mus = golden_inputs(name)
        out[name + "/kernel_grad"] = crf_fgrad_oracle.ref_full_kernel_grad(features, unary, p, G, mus)
    np.savez_compressed(os.path.join(HERE, GOLDEN), **out)


if __name__ == "__main__":
    main()
