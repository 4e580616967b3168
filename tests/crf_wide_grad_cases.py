"""Cases of the CRF gradient above 32 labels (test_crf_wide_grad_cpu.py, test_gpu_crf_wide_grad.py).

The truths and bars are crf_grad_cases.GradTruth's (Potts) and crf_compat_cases.CompatTruth's (matrices): the
label-chunked backward runs meanfield.cu's operation order for the slices, G_t and the mat-vecs (the float32 models'
arith="device"), and its sums stay inside those bars' floors.  A Potts weight's terms are added over a thread's four
labels, the block's 256 pixels (a tree of depth 8), the iterations, then the ceil(M/4) * ceil(N/256) blocks of the
image (8463 for one 81-label 321x321 image: 34 per thread, then a tree of depth 8), a depth below 80, so below 2^-18
of the sum of |S_k|·|Q_t| against the floor of 2^-16.  An entry of dL/dmu is summed over a 32-pixel slab, the chunk's
slabs (at most 202 at 321x321), the iterations and the 16 chunks, a depth below 270, so about 2^-16 of its sum
against the floor of 2^-14.
"""
import numpy as np

import helpers
from crf_compat_cases import compat_mats
from crf_grad_cases import grad_params, upstream

GOLDEN = "crf_wide_grad_ref.npz"
WIDE_GRAD_M = [33, 36, 81, 128, 255]   # phantom lanes in the last quad (3, 1) and whole quads
# the cases of the frozen reference results (tests/golden/make_crf_wide_grad_golden.py); the matrices are symmetric
# because the reference symmetrises: name -> (H, W, image, M, scale factor, T, seed, "potts" or "sym")
GOLDEN_CASES = {
    "potts_33": (9, 11, "noise", 33, 1.0, 4, 3, "potts"),
    "potts_81": (17, 19, "smooth", 81, 12.0, 3, 5, "potts"),
    "sym_33": (9, 11, "noise", 33, 12.0, 5, 7, "sym"),
    "sym_81": (17, 19, "smooth", 81, 1.0, 3, 9, "sym"),
}


def golden_inputs(name):
    """(image (H, W, 3), unary (H, W, M), G (H, W, M), params, (mu_bi, mu_sp) or None) of a golden case."""
    H, W, img, M, sf, T, seed, kind = GOLDEN_CASES[name]
    image = helpers.small_image(np.random.RandomState(seed), H, W, img)
    unary = helpers.log_unary(1, H, W, M, seed, scale=1.0)[0]
    mus = compat_mats(kind, M, seed) if kind != "potts" else None
    return image, unary, upstream(H, W, M, seed), grad_params(sf, T), mus
