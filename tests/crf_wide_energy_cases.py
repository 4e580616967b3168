"""Cases of the CRF energy above 32 labels (test_crf_wide_energy_cpu.py, test_gpu_crf_wide_energy.py,
tests/golden/make_crf_wide_energy_golden.py)."""
import numpy as np

import helpers
from crf_compat_cases import compat_mats
from crf_energy_cases import ENERGY_REL, q_of
from crf_fgrad_cases import features_of
from crf_grad_cases import grad_params

GOLDEN = "crf_wide_energy_ref.npz"
# name -> (q kind, M, image kind, bilateral "image" or a features_of kind, matrix kind or None, unary?)
GOLDEN_CASES = {
    "potts_image": ("random", 33, "photo", "image", None, True),
    "matrix_image": ("random", 40, "smooth", "image", "nonsym", True),
    "potts_features": ("random", 81, "photo", "guide", None, False),
    "matrix_features": ("softmax", 40, "noise", "random", "sym", True),
    "onehot_image": ("onehot", 81, "noise", "image", None, True),
}


def golden_inputs(name):
    """-> (q, unary or None, params, m (m_bi, m_sp) as MatrixCompatibility takes them or None, image, features or
    None) of one golden case on a 9x11 image, all (H, W, ...) float32 / uint8."""
    qk, M, img, bil, mk, with_u = GOLDEN_CASES[name]
    H, W = 9, 11
    image = helpers.small_image(np.random.RandomState(5), H, W, img)
    p = grad_params(4.0, 0)
    feats = None if bil == "image" else features_of(bil, image, p, 8)
    unary = helpers.log_unary(1, H, W, M, 6, scale=1.0)[0] if with_u else None
    return q_of(qk, H, W, M, 7), unary, p, (compat_mats(mk, M, 5) if mk else None), image, feats


# The device against the float64 restatement: |device - truth| <= energy_rel(M) * scale, scale the sum of the
# magnitudes behind the result (crf_energy_oracle).  Every float32 operation behind one value rounds once, by at most
# 2^-24 of the magnitudes it has summed so far, which the scale bounds.  Per value that is, at most:
#   FILTER_ROUNDINGS for the filter F(Q) (splat, d + 1 = 6 axis blurs of 3 terms, a 6-term slice: crf_energy_cases);
#   M for the message (mu F)_l, an fma chain over the labels (one product for Potts);
#   M for the per-pixel term sum_l q_l (mu F)_l, or for the transposed message of the gradient;
#   2 M for the gradient's running sum over both lattices' messages.
# The bar is that worst case, (FILTER_ROUNDINGS + 4 M) 2^-24, and never below the fused path's ENERGY_REL: at 81
# labels 2^-15.5, at 255 labels (each message 255 products) 2^-14.
FILTER_ROUNDINGS = 30


def energy_rel(M):
    return max(ENERGY_REL, (FILTER_ROUNDINGS + 4 * M) * 2.0 ** -24)


def check_terms(got, want, scale, M, what=""):
    got = np.asarray(got, np.float64)
    assert np.all(np.isfinite(got)), what
    err = np.abs(got - want)
    bar = energy_rel(M) * scale
    assert np.all(err <= bar + 1e-30), "%s terms %s want %s err %s bar %s" % (what, got, want, err, bar)


def check_grad(got, want, scale, M, what=""):
    got = np.asarray(got, np.float64)
    assert np.all(np.isfinite(got)), what
    excess = np.abs(got - want) / (energy_rel(M) * scale + 1e-30)
    assert excess.max() <= 1.0, "%s worst err/bar %g at %s" % (what, excess.max(), np.unravel_index(excess.argmax(),
                                                                                                      excess.shape))
    return float(excess.max())
