"""Regenerate tests/golden/crf_compat_grad_ref.npz: the reference CRF with MatrixCompatibility on both terms
(labelcompatibility.cpp:64-108; DenseCRF::inference and DenseCRF::gradient, built into
oracle/_ref/libdensecrf_compat_ref.so by oracle/compat.mk) on a few images, so that the compatibility tests have a pin
to the reference wherever oracle/_ref was not built.  Run from the repository root:
python tests/golden/make_crf_compat_golden.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.join(HERE, "..", ".."), os.path.join(HERE, "..")]

from crf_compat_cases import GOLDEN, GOLDEN_CASES, golden_inputs  # noqa: E402
from oracle import crf_compat_oracle  # noqa: E402


def main():
    if not crf_compat_oracle.ref_available():
        sys.exit("oracle/_ref/libdensecrf_compat_ref.so is not built")
    out = {}
    for name in GOLDEN_CASES:
        image, unary, G, p, mus = golden_inputs(name)
        q, gU, lg = crf_compat_oracle.ref_crf_compat(image, unary, p, mus[0], mus[1], G)
        out[name + "/q"] = q
        out[name + "/grad_unary"] = gU
        out[name + "/lbl_cmp_grad_sp"] = lg["sp"]
        out[name + "/lbl_cmp_grad_bi"] = lg["bi"]
    np.savez_compressed(os.path.join(HERE, GOLDEN), **out)


if __name__ == "__main__":
    main()
