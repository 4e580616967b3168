"""oracle/crf_fgrad_oracle.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The gradient of the dense CRF to caller-given bilateral features, per pixel: DenseKernel::featureGradient
(pairwise.cpp) for the kernel the reference's addPairwiseEnergy(features, PottsCompatibility(w1) or
MatrixCompatibility, DIAG_KERNEL, NORMALIZE_SYMMETRIC) adds at p = 1, restated in numpy.  It is crf_kgrad_oracle's
derivation stopped before the reduction: with x_t = -mu^T g_{t+1} and c = sum_t 1/2 n^3 sum_l (x_t K(n Q_t) +
K^T(n x_t) Q_t),

    dL/df = sum_t d^K <n x_t, K (n Q_t)>  -  d^K <c, K 1>      (N, 5), one row per pixel

and sum_pixels f_i (dL/df)_i is the kernel's DIAG dL/dp_i (crf_kgrad_oracle.theta_grad's dp).  The spatial kernel
stays the one of params (theta_gamma), and its dL/dtheta_gamma comes out beside.

``FeatProblem`` is a meanfield64.Problem whose bilateral lattice is the oracle's lattice (crf_oracle.OracleLattice,
pinned to permutohedral.cpp) of the given float32 features.  ``Frozen`` holds every pixel's simplex: its
``frozen_problem(f)`` recomputes the barycentric weights in float64 from perturbed features, the forward the
derivative is exact for, for central finite differences.  ``convention="reference"`` is the reference's K^T
(crf_kgrad_oracle); the float32 ``dtype`` with meanfield64's ``splat_order`` / ``arith`` switches models the device's
rounding; ``mutant`` takes crf_kgrad_oracle.MUTANTS.

``ref_full_kernel_grad`` is the reference's own kernel_grad for a term added as addPairwiseEnergy(features, ...,
FULL_KERNEL) at P = I: fg f^T, with fg its featureGradient, built by oracle/fgrad.mk into
_ref/libdensecrf_fgrad_ref.so (when the reference is present; the built .so travels with the tree).

Only tests/ may import this module.
"""
import ctypes as C
import copy
import os
import subprocess

import numpy as np

from . import crf_compat_oracle, crf_grad_oracle, crf_oracle, meanfield64
from . import crf_kgrad_oracle as K

MUTANTS = K.MUTANTS

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_ref", "libdensecrf_fgrad_ref.so")
_REF = None


def build(force=False):
    if os.path.exists("/root/reference/CRF/src/densecrf.cpp") and (force or not os.path.exists(_SO)):
        subprocess.check_call(["make", "-C", _HERE, "-f", "fgrad.mk", "ref"], stdout=subprocess.DEVNULL)


def ref_available():
    return os.path.exists(_SO)


def ref_full_kernel_grad(features, unary, params, grad_q, mus=None):
    """The reference's kernel_grad for its DenseCRFWrapper Gaussian term (params' theta_gamma, w2 or mu_sp) and a term
    addPairwiseEnergy(features, PottsCompatibility(w1) or MatrixCompatibility(mu_bi), FULL_KERNEL) at P = I:
    features (H, W, 5) float32, unary (H, W, M) the values CRF() takes, grad_q (H, W, M).  -> (27,) float32: the
    Gaussian term's dL/dp (x, y), then dL/dP (5 x 5) column-major."""
    global _REF
    if _REF is None:
        R = C.CDLL(_SO)
        f32p = crf_oracle._f32p
        R.ref_densecrf_fgrad.argtypes = ([C.c_int] * 3 + [f32p, C.c_float, C.c_void_p, f32p, C.c_float, C.c_void_p]
                                         + [C.c_float] * 2 + [C.c_int, f32p, f32p])
        _REF = R
    H, W, M = unary.shape
    out = np.zeros(27, np.float32)
    f = lambda m: np.ascontiguousarray(m, np.float32).ravel()
    keep = [] if mus is None else [f(mus[0]), f(mus[1])]
    ptr = lambda i: None if mus is None else keep[i].ctypes.data_as(C.c_void_p)
    p = params
    _REF.ref_densecrf_fgrad(W, H, M, f(-unary), p.w1, ptr(0), f(features), p.w2, ptr(1), p.theta_gamma_x,
                            p.theta_gamma_y, int(p.n_iters), f(grad_q), out)
    return out


def full_kernel_grad(df, features):
    """dL/dP (25,) at P = I in the reference's order (Eigen column-major fg f^T) from dL/df (N, 5)."""
    return (np.asarray(df, np.float64).T @ np.asarray(features, np.float64).reshape(-1, 5)).ravel(order="F")


def image_features(image, params):
    """The image path's float32 bilateral features (H, W, 5): float32(x)/theta_alpha_x, ..., b/theta_beta_b as the
    lattice build divides them."""
    sig = np.asarray([params.theta_alpha_x, params.theta_alpha_y, params.theta_beta_r, params.theta_beta_g,
                      params.theta_beta_b], np.float32)
    raw = K._raw_features(image, 5).astype(np.float32)
    return (raw / sig).astype(np.float32).reshape(image.shape[0], image.shape[1], 5)


def simplex(f):
    """crf_kgrad_oracle.simplex on given float32 features (N, d): -> (rank, rem0 float64, bary float32)."""
    d = f.shape[1]
    el = K._elevate(np.asarray(f, np.float32), K._scales(d, np.float32))
    inv = np.float32(1.0) / np.float32(d + 1)
    v = np.rint(inv * el)
    rem0 = (v * np.float32(d + 1)).astype(np.float32)
    isum = v.astype(np.int64).sum(1)
    rank = np.zeros(el.shape, np.int64)
    for i in range(d):
        di = el[:, i] - rem0[:, i]
        for j in range(i + 1, d + 1):
            c = di < el[:, j] - rem0[:, j]
            rank[:, i] += c
            rank[:, j] += ~c
    rank += isum[:, None]
    lo, hi = rank < 0, rank >= d + 1
    rank[lo] += d + 1
    rank[hi] -= d + 1
    rem0 = rem0 + np.float32(d + 1) * lo.astype(np.float32) - np.float32(d + 1) * hi.astype(np.float32)
    vv = ((el - rem0) * inv).astype(np.float32)
    bc = np.zeros((el.shape[0], d + 2), np.float32)
    rows = np.arange(el.shape[0])
    for i in range(d + 1):
        p = d - rank[:, i]
        bc[rows, p] += vv[:, i]
        bc[rows, p + 1] -= vv[:, i]
    bc[:, 0] += np.float32(1.0) + bc[:, d + 1]
    return rank, rem0.astype(np.float64), bc[:, :d + 1]


class FeatProblem(meanfield64.Problem):
    """meanfield64.Problem with the bilateral lattice built on `features` (H, W, 5) float32; params gives the spatial
    sigmas, the weights and the iterations."""

    def __init__(self, features, params):
        H, W = features.shape[:2]
        super().__init__(np.zeros((H, W, 3), np.uint8), params)
        self.features = np.ascontiguousarray(features, np.float32).reshape(H * W, 5)
        self.params = params
        self.lattices[1] = meanfield64.Lattice(crf_oracle.OracleLattice(self.features), params.w1)


class Frozen(object):
    """A FeatProblem with every pixel's bilateral simplex held: barycentric weights as a function of the features."""

    def __init__(self, problem):
        self.problem = problem
        self.f32 = problem.features
        self.rank, self.rem0, bary32 = simplex(self.f32)
        if not np.array_equal(bary32, problem.lattices[1].bary):
            raise AssertionError("the restated simplex does not reproduce the feature lattice's barycentric weights")
        # the spatial lattice, held as crf_kgrad_oracle.Frozen holds it
        zero = np.zeros((problem.H, problem.W, 3), np.uint8)
        self.theta_sp = np.array([problem.params.theta_gamma_x, problem.params.theta_gamma_y], np.float64)
        self.sp_rank, self.sp_rem0, sp32 = K.simplex(zero, self.theta_sp)
        if not np.array_equal(sp32, problem.lattices[0].bary):
            raise AssertionError("the restated simplex does not reproduce the spatial lattice's barycentric weights")
        self.sp_f = K._raw_features(zero, 2) / self.theta_sp

    @staticmethod
    def _bary(f, rank, rem0):
        """float64 barycentric weights of features f (N, d) on the held simplices (rank, rem0)."""
        d = f.shape[1]
        el = K._elevate(np.asarray(f, np.float64), K._scales(d, np.float64))
        v = (el - rem0) / (d + 1)
        rows = np.arange(el.shape[0])[:, None]
        rho = np.empty_like(rank)
        rho[rows, d - rank] = np.arange(d + 1)[None, :]
        vr = v[rows, rho]
        b = vr - np.roll(vr, 1, axis=1)
        b[:, 0] += 1.0
        return b

    def frozen_problem(self, f):
        """A copy of the problem whose lattices carry the float64 weights: the bilateral one at features f (N, 5),
        the spatial one at the problem's theta_gamma."""
        P = copy.copy(self.problem)
        P._norms = {}
        P.lattices = []
        for L, bary in ((self.problem.lattices[0], self._bary(self.sp_f, self.sp_rank, self.sp_rem0)),
                        (self.problem.lattices[1], self._bary(f, self.rank, self.rem0))):
            L2 = copy.copy(L)
            L2.bary = bary
            P.lattices.append(L2)
        return P


def feature_grad(fz, unary, grad_q, mus=None, convention="exact", mutant=None, dtype=np.float64,
                 splat_order=None, arith="oracle", exp_seed=0):
    """For L = <grad_q, Q_T> on the frozen lattices at the problem's own features: -> (df (N, 5) = dL/df per pixel,
    dtheta_sp (2,) = dL/d{theta_gamma_x, theta_gamma_y}, mag (N, 5) = the magnitude of df's terms before they cancel).

    float64: the truth.  float32: a model of the device's rounding (as crf_kgrad_oracle.theta_grad)."""
    f64 = dtype == np.float64
    T = fz.problem.n_iters
    P = fz.frozen_problem(fz.f32.astype(np.float64)) if f64 else fz.problem
    M = grad_q.shape[-1]
    if mus is None:
        Qs = P.run(unary, T, dtype, splat_order, arith, exp_seed=exp_seed)
    else:
        Qs = crf_compat_oracle.run(P, unary, mus, T, dtype, splat_order, arith, exp_seed)
    Qs = [q.reshape(P.N, M).astype(dtype) for q in Qs]
    G = np.asarray(grad_q, np.float64).reshape(P.N, M).astype(dtype)
    norms = P.norms(dtype, None if f64 else splat_order)
    mu = K._mus(P, mus)
    for k, L in enumerate(P.lattices):
        mu[k] = (-L.w * np.eye(M) if mu[k] is None else mu[k]).astype(dtype)
    fwd, rev = (K.L_blur_fwd, K.L_blur_rev) if convention == "exact" else (K.L_blur_rev, K.L_blur_fwd)
    if mutant == "forward_order":
        fwd = rev = K.L_blur_fwd
    ranks = [fz.sp_rank, fz.rank]
    S = [L.splat_matrix(L.bary, dtype, None if f64 else splat_order) for L in P.lattices]
    alpha = [L.alpha(dtype) for L in P.lattices]
    df = [np.zeros((P.N, L.d), dtype) for L in P.lattices]
    mag = [np.zeros((P.N, L.d)) for L in P.lattices]
    csum = [np.zeros(P.N, dtype) for _ in P.lattices]

    def vjp(q, gt):
        return q * (gt - (gt * q).sum(1)[:, None])

    g = vjp(Qs[T], G)
    for t in range(T - 1, -1, -1):
        Gt = np.zeros((P.N, M), dtype)
        for k, L in enumerate(P.lattices):
            n = norms[k][:, None]
            x = -(g @ mu[k])
            y = Qs[t]
            vy, vx = fwd(L, S[k] @ (n * y)), rev(L, S[k] @ (n * x))
            s = ((n * x)[:, None, :] * vy[L.offset]).sum(2) + ((n * y)[:, None, :] * vx[L.offset]).sum(2)
            df[k] += alpha[k] * K._rot(L, s, ranks[k], mutant)
            mag[k] += float(alpha[k]) * K._rot(L, s.astype(np.float64), ranks[k], magnitude=True)
            kny = L.slice(L.blur(S[k] @ (n * y), False), False)
            ktnx = L.slice(crf_grad_oracle.blur_t(L, S[k] @ (n * x)), False)
            csum[k] += dtype(0.5) * norms[k] ** 3 * (x * kny + ktnx * y).sum(1)
            Gt -= (L.slice(crf_grad_oracle.blur_t(L, S[k] @ (n * g)), False) * n) @ mu[k]
        g = vjp(Qs[t], Gt)
    for k, L in enumerate(P.lattices):
        if T > 0 and mutant != "no_norm":
            v1 = fwd(L, S[k] @ np.ones((P.N, 1), dtype))[:, 0]
            vc = rev(L, S[k] @ csum[k][:, None])[:, 0]
            s = csum[k][:, None] * v1[L.offset] + vc[L.offset]
            df[k] -= alpha[k] * K._rot(L, s, ranks[k], mutant)
            mag[k] += float(alpha[k]) * K._rot(L, s.astype(np.float64), ranks[k], magnitude=True)
    f_sp = fz.sp_f if f64 else fz.sp_f.astype(np.float32)
    dp_sp = (f_sp * df[0]).sum(0, dtype=dtype).astype(np.float64)
    return df[1].astype(np.float64), -dp_sp / fz.theta_sp, mag[1]


def loss(P, unary, G, T, mus=None):
    return K.loss(P, unary, G, T, mus)


def finite_diff(fz, unary, grad_q, direction, mus=None, h=1e-4):
    """Central difference of <grad_q, Q_T> on the frozen lattices along `direction` (N, 5) of the features."""
    G = np.asarray(grad_q, np.float64)
    f0 = fz.f32.astype(np.float64)
    T = fz.problem.n_iters
    return (loss(fz.frozen_problem(f0 + h * direction), unary, G, T, mus)
            - loss(fz.frozen_problem(f0 - h * direction), unary, G, T, mus)) / (2 * h)
