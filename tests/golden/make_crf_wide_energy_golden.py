"""tests/golden/make_crf_wide_energy_golden.py -- regenerates tests/golden/crf_wide_energy_ref.npz.

Runs ONLY where the reference is present: builds oracle/_ref/libdensecrf_energy_ref.so (oracle/energy.mk, the
reference's own CRF sources around DenseCRF::klDivergence, which take any label count) and stores, per case of
tests/crf_wide_energy_cases.py (33, 40 and 81 labels), the reference's four terms (entropy, unary, spatial,
bilateral), separated as tests/golden/make_crf_energy_golden.py separates them.  The inputs are regenerated from their
seeds by the cases module.

usage: python tests/golden/make_crf_wide_energy_golden.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))                    # tests/
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))   # the repository

from crf_wide_energy_cases import GOLDEN, GOLDEN_CASES, golden_inputs   # noqa: E402
from oracle import crf_energy_oracle as E   # noqa: E402


def main():
    E.build(force=True)
    assert E.ref_available(), "the reference build is missing"
    out = {}
    for name in GOLDEN_CASES:
        q, unary, p, m, image, feats = golden_inputs(name)
        out[name + "/terms"] = E.ref_terms(q, unary, p, m, image=image, features=feats)
        print(name, out[name + "/terms"])
    np.savez(os.path.join(HERE, GOLDEN), **out)


if __name__ == "__main__":
    main()
