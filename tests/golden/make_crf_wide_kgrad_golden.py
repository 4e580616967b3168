"""Regenerate tests/golden/crf_wide_kgrad_ref.npz: the reference's own kernel_grad above 32 labels, for the image
path's DIAG kernels (oracle/kgrad.mk) and for a caller-given FULL_KERNEL term at P = I (oracle/fgrad.mk), with Potts
and MatrixCompatibility terms, so that the label-chunked kernel-bandwidth and feature tests have a pin to the
reference wherever oracle/_ref was not built.  Run from the repository root:
python tests/golden/make_crf_wide_kgrad_golden.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.join(HERE, "..", ".."), os.path.join(HERE, "..")]

from crf_wide_kgrad_cases import GOLDEN, GOLDEN_CASES, golden_inputs  # noqa: E402
from oracle import crf_fgrad_oracle, crf_kgrad_oracle  # noqa: E402


def main():
    if not (crf_kgrad_oracle.ref_available() and crf_fgrad_oracle.ref_available()):
        sys.exit("oracle/_ref/libdensecrf_kgrad_ref.so or libdensecrf_fgrad_ref.so is not built")
    out = {}
    for name in GOLDEN_CASES:
        image, feats, unary, G, p, mus, kind = golden_inputs(name)
        if kind == "theta":
            out[name + "/kernel_grad"] = crf_kgrad_oracle.ref_kernel_grad(image, unary, p, G, mus)
        else:
            out[name + "/kernel_grad"] = crf_fgrad_oracle.ref_full_kernel_grad(feats, unary, p, G, mus)
    np.savez_compressed(os.path.join(HERE, GOLDEN), **out)


if __name__ == "__main__":
    main()
