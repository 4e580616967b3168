"""oracle/crf_energy_oracle.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The dense CRF's energy of given marginals (DenseCRF::klDivergence, densecrf.cpp:213-235) and its gradient, restated in
float64 numpy on a meanfield64.Problem's lattices (crf_fgrad_oracle.FeatProblem for caller-given features).  With
F_k(Q) = n_k K_k(n_k Q) per kernel (lattice order: spatial, bilateral) and the library's matrices (Potts mu = -w I,
the reference's MatrixCompatibility(m) mu = (m + m^T) / 2):

    terms = (sum Q log max(Q, 1e-20f), -sum unary Q, sum Q . mu_sp F_sp(Q), sum Q . mu_bi F_bi(Q))
    d/dQ  = g0 (Q > 1e-20f ? log Q + 1 : log 1e-20f) - g1 unary + sum_k g_k (mu_k F_k(Q) + mu_k^T F_k^T(Q))
    d/dunary = -g1 Q

F^T is the transposed blur (crf_grad_oracle.blur_t: the axes d..0), as the device differentiates its own K.  Each
function also returns the sum of the magnitudes behind each result (|Q| |mu| F(Q) with F >= 0 for Q >= 0, and so
on), the scale of a float32 computation's rounding error.

``ref_kl`` is the reference's own klDivergence with nothing, the unary alone or one pairwise term alone, built by
oracle/energy.mk into _ref/libdensecrf_energy_ref.so when the reference is present; ``ref_terms`` separates the four
terms from those.  tests/golden/make_crf_energy_golden.py freezes them: the tests never need the reference.

Only tests/ may import this module.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from . import crf_grad_oracle, crf_oracle

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_ref", "libdensecrf_energy_ref.so")
_REF = None
EPS = float(np.float32(1e-20))   # the reference's 1e-20f


def build(force=False):
    if os.path.exists("/root/reference/CRF/src/densecrf.cpp") and (force or not os.path.exists(_SO)):
        subprocess.check_call(["make", "-C", _HERE, "-f", "energy.mk", "ref"], stdout=subprocess.DEVNULL)


def ref_available():
    return os.path.exists(_SO)


def ref_kl(q, term, unary=None, w=0.0, mu=None, sigmas=None, image=None, features=None):
    """The reference's klDivergence of q (H, W, M) for a DenseCRF2D with, by `term`: 0 nothing, 1 the unary (the
    values CRF() takes, so the energy -unary), 2 addPairwiseGaussian(sigmas[0:2]), 3 addPairwiseBilateral(sigmas[0:5],
    image), 4 addPairwiseEnergy(features (H, W, 5)); each pairwise term with MatrixCompatibility(mu) or, mu None,
    PottsCompatibility(w)."""
    global _REF
    if _REF is None:
        R = C.CDLL(_SO)
        R.ref_densecrf_kl.restype = C.c_double
        R.ref_densecrf_kl.argtypes = [C.c_int] * 3 + [C.c_void_p, C.c_int, C.c_void_p, C.c_float] + [C.c_void_p] * 4
        _REF = R
    H, W, M = q.shape
    keep = []

    def ptr(a, dtype=np.float32):
        if a is None:
            return None
        a = np.ascontiguousarray(a, dtype)
        keep.append(a)
        return a.ctypes.data_as(C.c_void_p)

    return float(_REF.ref_densecrf_kl(W, H, M, ptr(q), int(term), ptr(None if unary is None else -unary), float(w),
                                      ptr(mu), ptr(sigmas), ptr(image, np.uint8), ptr(features)))


def ref_terms(q, unary, params, mus=None, image=None, features=None):
    """(4,) float64: the reference's entropy, unary, spatial and bilateral terms of q (H, W, M), each pairwise one the
    difference of klDivergence with that term alone and with none.  mus = (m_bi, m_sp) as MatrixCompatibility takes
    them, or None for PottsCompatibility(w1 / w2); image (H, W, 3) or features (H, W, 5)."""
    p = params
    e = ref_kl(q, 0)
    u = 0.0 if unary is None else ref_kl(q, 1, unary) - e
    m_bi, m_sp = (None, None) if mus is None else mus
    sp = ref_kl(q, 2, w=p.w2, mu=m_sp, sigmas=[p.theta_gamma_x, p.theta_gamma_y]) - e
    if features is None:
        bi = ref_kl(q, 3, w=p.w1, mu=m_bi, image=image,
                    sigmas=[p.theta_alpha_x, p.theta_alpha_y, p.theta_beta_r, p.theta_beta_g, p.theta_beta_b])
    else:
        bi = ref_kl(q, 4, w=p.w1, mu=m_bi, features=features)
    return np.array([e, u, sp, bi - e])


def _mus(problem, mus, M):
    """[mu_sp, mu_bi] float64 in lattice order from mus = (mu_bi, mu_sp) in the library's convention, or Potts."""
    if mus is None:
        return [-L.w * np.eye(M) for L in problem.lattices]
    return [np.asarray(mus[1], np.float64), np.asarray(mus[0], np.float64)]


def filt(problem, k, Q, transpose=False):
    """F_k(Q) = n K(n Q) of lattice k for Q (N, M) float64, or F_k^T(Q) = n K^T(n Q) with `transpose`."""
    L, n = problem.lattices[k], problem.norms(np.float64)[k]
    if not transpose:
        return L.filter(Q * n[:, None], np.float64) * n[:, None]
    v = L.splat_matrix(L.bary, np.float64, None) @ (Q * n[:, None])
    return L.slice(crf_grad_oracle.blur_t(L, v), False) * n[:, None]


def _flat(a, N, M):
    return None if a is None else np.asarray(a, np.float64).reshape(N, M)


def terms(problem, q, unary=None, mus=None):
    """q, unary (H, W, M) -> (terms (4,), scale (4,)) in float64."""
    N = problem.N
    M = q.shape[-1]
    Q, U = _flat(q, N, M), _flat(unary, N, M)
    lq = np.log(np.maximum(Q, EPS))
    t = np.zeros(4)
    s = np.zeros(4)
    t[0], s[0] = (Q * lq).sum(), np.abs(Q * lq).sum()
    if U is not None:
        t[1], s[1] = -(U * Q).sum(), np.abs(U * Q).sum()
    for k, mu in enumerate(_mus(problem, mus, M)):
        F = filt(problem, k, Q)
        t[2 + k] = (Q * (F @ mu.T)).sum()
        s[2 + k] = (np.abs(Q) * (np.abs(F) @ np.abs(mu).T)).sum()
    return t, s


def gradient(problem, q, unary, grad_terms, mus=None):
    """d(grad_terms . terms) -> (dq (H, W, M), dunary (H, W, M), scale (H, W, M)) in float64, scale the magnitude sum
    behind each element of dq."""
    N = problem.N
    H, W, M = q.shape
    Q, U = _flat(q, N, M), _flat(unary, N, M)
    g = np.asarray(grad_terms, np.float64)
    lq = np.log(np.maximum(Q, EPS))
    d0 = np.where(Q > EPS, lq + 1.0, lq)
    dq = g[0] * d0
    sc = np.abs(g[0] * d0)
    if U is not None:
        dq = dq - g[1] * U
        sc = sc + np.abs(g[1] * U)
    for k, mu in enumerate(_mus(problem, mus, M)):
        F, Ft = filt(problem, k, Q), filt(problem, k, Q, transpose=True)
        dq = dq + g[2 + k] * (F @ mu.T + Ft @ mu)
        sc = sc + abs(g[2 + k]) * (np.abs(F) @ np.abs(mu).T + np.abs(Ft) @ np.abs(mu))
    return dq.reshape(H, W, M), (-g[1] * Q).reshape(H, W, M), sc.reshape(H, W, M)


def energy_of(problem, q, unary, grad_terms, mus=None):
    """grad_terms . terms: the scalar whose gradient ``gradient`` is (for finite differences)."""
    return float(np.dot(np.asarray(grad_terms, np.float64), terms(problem, q, unary, mus)[0]))
