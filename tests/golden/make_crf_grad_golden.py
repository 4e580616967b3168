"""Regenerate tests/golden/crf_grad_ref.npz: the reference's own DenseCRF::gradient (densecrf.cpp:238-297, built into
oracle/_ref/libdensecrf_grad_ref.so by oracle/grad.mk) on a few images, so that the gradient tests have a pin to the
reference wherever oracle/_ref was not built.  Run from the repository root: python tests/golden/make_crf_grad_golden.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.join(HERE, "..", ".."), os.path.join(HERE, "..")]

from crf_grad_cases import GOLDEN, GOLDEN_CASES, golden_inputs  # noqa: E402
from oracle import crf_grad_oracle  # noqa: E402


def main():
    if not crf_grad_oracle.ref_available():
        sys.exit("oracle/_ref/libdensecrf_grad_ref.so is not built")
    out = {}
    for name in GOLDEN_CASES:
        image, unary, G, p = golden_inputs(name)
        gU, gw = crf_grad_oracle.ref_crf_gradient(image, unary, p, G)
        out[name + "/grad_unary"] = gU
        out[name + "/grad_potts"] = np.array(gw, np.float64)
    np.savez_compressed(os.path.join(HERE, GOLDEN), **out)


if __name__ == "__main__":
    main()
