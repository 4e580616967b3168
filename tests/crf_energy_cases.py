"""Cases of the CRF energy (test_crf_energy_cpu.py, test_gpu_crf_energy.py, tests/golden/make_crf_energy_golden.py)."""
import numpy as np

import helpers
from crf_compat_cases import compat_mats
from crf_fgrad_cases import features_of
from crf_grad_cases import grad_params
from oracle import crf_energy_oracle as E
from oracle import crf_fgrad_oracle, meanfield64

# The device's terms and gradients against the float64 restatement: |device - truth| <= ENERGY_REL * scale, scale the
# sum of the magnitudes behind the result (crf_energy_oracle: |Q| |mu| F(Q) ...).  Each product and each of the
# splat's, blur's and slice's additions rounds once in float32 (2^-24 relative); a pixel's message passes through at
# most about 30 of them (d + 1 = 6 axis blurs of 3 terms, a 6-term slice, the norm's own splat-blur-slice), so its
# relative error stays below 2^-19, and the double per-block sums add nothing visible.  2^-16 leaves 8x over that.
ENERGY_REL = 2.0 ** -16
GOLDEN = "crf_energy_ref.npz"
# name -> (q kind, M, image kind, bilateral "image" or a features_of kind, matrix kind or None, unary?)
GOLDEN_CASES = {
    "potts_image": ("random", 4, "photo", "image", None, True),
    "matrix_image": ("random", 5, "smooth", "image", "nonsym", True),
    "potts_features": ("random", 3, "photo", "guide", None, False),
    "matrix_features": ("softmax", 6, "noise", "random", "sym", True),
    "onehot_image": ("onehot", 21, "noise", "image", None, True),
}


def q_of(kind, H, W, M, seed):
    """(H, W, M) float32 non-negative q: "random" positive and unnormalised with exact zeros and values below 1e-20,
    "softmax" marginals, "onehot" a label map."""
    rng = np.random.RandomState(seed)
    if kind == "onehot":
        return np.eye(M, dtype=np.float32)[rng.randint(0, M, (H, W))]
    if kind == "softmax":
        x = rng.randn(H, W, M) * 2.0
        e = np.exp(x - x.max(-1, keepdims=True))
        return (e / e.sum(-1, keepdims=True)).astype(np.float32)
    q = rng.uniform(0.0, 1.5, (H, W, M))
    q[rng.rand(H, W, M) < 0.1] = 0.0
    q[rng.rand(H, W, M) < 0.03] = 1e-25
    return q.astype(np.float32)


def golden_inputs(name):
    """-> (q, unary or None, params, m (m_bi, m_sp) as MatrixCompatibility takes them or None, image, features or
    None) of one golden case, all (H, W, ...) float32 / uint8."""
    qk, M, img, bil, mk, with_u = GOLDEN_CASES[name]
    H, W = 9, 11
    image = helpers.small_image(np.random.RandomState(5), H, W, img)
    p = grad_params(4.0, 0)
    feats = None if bil == "image" else features_of(bil, image, p, 8)
    unary = helpers.log_unary(1, H, W, M, 6, scale=1.0)[0] if with_u else None
    return q_of(qk, H, W, M, 7), unary, p, (compat_mats(mk, M, 5) if mk else None), image, feats


def library_mus(m):
    """The library's (mu_bi, mu_sp) of the reference's MatrixCompatibility(m): (m + m^T) / 2."""
    return None if m is None else tuple(0.5 * (x.astype(np.float64) + x.astype(np.float64).T) for x in m)


def problem(image, params, features=None):
    return meanfield64.Problem(image, params) if features is None else crf_fgrad_oracle.FeatProblem(features, params)


def check_terms(got, want, scale, what=""):
    got = np.asarray(got, np.float64)
    assert np.all(np.isfinite(got)), what
    err = np.abs(got - want)
    assert np.all(err <= ENERGY_REL * scale + 1e-30), "%s terms %s want %s err %s bar %s" % (
        what, got, want, err, ENERGY_REL * scale)


def check_grad(got, want, scale, what=""):
    got = np.asarray(got, np.float64)
    assert np.all(np.isfinite(got)), what
    excess = np.abs(got - want) / (ENERGY_REL * scale + 1e-30)
    assert excess.max() <= 1.0, "%s worst err/bar %g at %s" % (what, excess.max(), np.unravel_index(excess.argmax(),
                                                                                                      excess.shape))
    return float(excess.max())


def grad_terms(B, seed):
    """(B, 4) float32 upstream gradients with every sign."""
    return np.random.RandomState(seed).uniform(-2.0, 2.0, (B, 4)).astype(np.float32)
