"""oracle/crf_kgrad_oracle.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The kernel-bandwidth gradient of the dense CRF (DenseCRF::gradient's kernel_grad, densecrf.cpp:238-297, under
DIAG_KERNEL and NORMALIZE_SYMMETRIC, pairwise.cpp:87-97 and :175-185) restated in numpy on a meanfield64.Problem's
lattices.  Per kernel k (lattice order: spatial, bilateral), with F_k(X) = n_k K_k(n_k X), n_k = (K_k 1 + 1e-20)^-1/2
and the forward t_{t+1} = U - mu_sp F_sp(Q_t) - mu_bi F_bi(Q_t) (Potts: mu = -w I):

    dL/df_k = sum_t  d^K <n x_t, K (n Q_t)>  -  d^K <c, K 1>,   x_t = -mu_k^T g_{t+1},
    c = sum_t 1/2 n^3 sum_labels (x_t K(n Q_t) + K^T(n x_t) Q_t)

d^K <a, K b> is the derivative through the barycentric weights with simplices, vertices and neighbours held
(Permutohedral::gradient, permutohedral.cpp:612-695): a·(B S b) + b·(B^T S a) at each pixel's d+1 vertices, rotated
by the pixel's simplex ranks and taken back through the elevation matrix.  Then, with f_k = raw / theta_k,
dL/dp_i = sum_pixels f_i (dL/df)_i (DIAG parameter p at 1, pairwise.cpp:178-179) and dL/dtheta_i = -dL/dp_i / theta_i.

``convention="reference"`` is what the reference computes: its Permutohedral::gradient(df, a, b) splats `a` and
blurs it in K's order before dotting with `b` (and the reverse), which is d<b, K a> = d<a, K^T b>; featureGradient
calls it as kernelGradient(a n, b n) and kernelGradient(c, ones).  So it differentiates K^T where K is meant: the
two differ wherever a blur neighbour is missing (the axis blurs then do not commute).

``ref_kernel_grad`` is the reference's own kernel_grad (Potts or MatrixCompatibility), built by oracle/kgrad.mk into
_ref/libdensecrf_kgrad_ref.so (when the reference is present; the built .so travels with the tree).

``frozen_problem`` is the forward the derivative is exact for: barycentric weights recomputed in float64 from
perturbed sigmas with every pixel's ranks and remainder-0 vertex (so offsets and neighbours) held, for central
finite differences.

Only tests/ may import this module.
"""
import copy
import ctypes as C
import os
import subprocess

import numpy as np

from . import crf_compat_oracle, crf_grad_oracle, crf_oracle

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_ref", "libdensecrf_kgrad_ref.so")
_REF = None

# name -> what the backward then does wrong
MUTANTS = {
    "no_norm": "the normalisation term -d<c, K 1> left out",
    "forward_order": "both directions blurred in K's axis order (B S where B^T S belongs)",
    "rank_off_by_one": "the rank rotation pairs vertex r0 with r0 + 2 instead of r0 + 1",
}

# theta order of dsrg_crf_params / grad_theta: alpha_x, alpha_y, beta_r, beta_g, beta_b, gamma_x, gamma_y
THETA_NAMES = ("theta_alpha_x", "theta_alpha_y", "theta_beta_r", "theta_beta_g", "theta_beta_b", "theta_gamma_x",
               "theta_gamma_y")


def build(force=False):
    if os.path.exists("/root/reference/CRF/src/densecrf.cpp") and (force or not os.path.exists(_SO)):
        subprocess.check_call(["make", "-C", _HERE, "-f", "kgrad.mk", "ref"], stdout=subprocess.DEVNULL)


def ref_available():
    return os.path.exists(_SO)


def ref_kernel_grad(image, unary, params, grad_q, mus=None):
    """The reference's DenseCRF::gradient kernel_grad for the CRF DenseCRFWrapper builds with `params`' sigmas and
    n_iters and Potts weights, or MatrixCompatibility(mu_bi), MatrixCompatibility(mu_sp) for mus = (mu_bi, mu_sp):
    image (H, W, 3) uint8, unary (H, W, M) the values CRF() takes, grad_q (H, W, M) = dL/dQ_T.  -> (7,) float32 dL/dp
    in the reference's order: spatial x, y, then bilateral x, y, r, g, b."""
    global _REF
    if _REF is None:
        R = C.CDLL(_SO)
        f32p, u8p = crf_oracle._f32p, crf_oracle._u8p
        R.ref_densecrf_kgrad.argtypes = ([C.c_int] * 3 + [f32p, C.c_float, C.c_void_p] + [C.c_float] * 6
                                         + [C.c_void_p] + [C.c_float] * 2 + [u8p, C.c_int, f32p, f32p])
        _REF = R
    H, W, M = unary.shape
    out = np.zeros(7, np.float32)
    f = lambda m: np.ascontiguousarray(m, np.float32).ravel()
    keep = [] if mus is None else [f(mus[0]), f(mus[1])]
    ptr = lambda i: None if mus is None else keep[i].ctypes.data_as(C.c_void_p)
    p = params
    _REF.ref_densecrf_kgrad(W, H, M, f(-unary), p.w1, ptr(0), p.theta_alpha_x, p.theta_alpha_y, p.theta_beta_r,
                            p.theta_beta_g, p.theta_beta_b, p.w2, ptr(1), p.theta_gamma_x, p.theta_gamma_y,
                            np.ascontiguousarray(image, np.uint8).ravel(), int(p.n_iters), f(grad_q), out)
    return out


def p_in_reference_order(dp):
    """dL/dp (7,) in dsrg_crf_params' theta order -> the reference's kernel_grad order (spatial first)."""
    return np.concatenate([dp[5:7], dp[0:5]])


def theta_of(params):
    return np.array([float(getattr(params, n)) for n in THETA_NAMES])


def _raw_features(image, d):
    H, W = image.shape[:2]
    y, x = np.mgrid[0:H, 0:W]
    cols = [x.ravel(), y.ravel()]
    if d == 5:
        cols += [image[..., c].ravel() for c in range(3)]
    return np.stack(cols, 1).astype(np.float64)         # (N, d) x, y[, r, g, b]


def _scales(d, dtype):
    inv = np.float32(np.sqrt(2.0 / 3.0) * (d + 1))      # permutohedral.cpp:179-182 (float inv_std_dev)
    s = np.array([1.0 / np.sqrt((i + 2) * (i + 1)) * float(inv) for i in range(d)])
    return s.astype(np.float32) if dtype == np.float32 else s


def _elevate(f, scale):
    """(N, d) features -> (N, d+1) elevated (permutohedral.cpp:201-207), in f's dtype, op by op."""
    N, d = f.shape
    el = np.zeros((N, d + 1), f.dtype)
    sm = np.zeros(N, f.dtype)
    for j in range(d, 0, -1):
        cf = f[:, j - 1] * scale[j - 1]
        el[:, j] = sm - f.dtype.type(j) * cf
        sm = sm + cf
    el[:, 0] = sm
    return el


def simplex(image, sigmas):
    """The float32 build's simplex of every pixel (permutohedral.cpp:191-242, lattice.cu:k_lattice_insert):
    -> (rank (N, d+1) int, rem0 (N, d+1) float64, bary (N, d+1) float32 as the build computes it)."""
    d = len(sigmas)
    f = (_raw_features(image, d).astype(np.float32) / np.asarray(sigmas, np.float32)).astype(np.float32)
    el = _elevate(f, _scales(d, np.float32))
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


class Frozen(object):
    """One image's lattices with every pixel's simplex held: barycentric weights as a function of the sigmas."""

    def __init__(self, problem, image, params):
        self.problem = problem
        th = theta_of(params)
        self.theta0 = th
        self.sig = [th[5:7], th[0:5]]                    # lattice order: spatial, bilateral
        self.raw, self.rank, self.rem0 = [], [], []
        for k, L in enumerate(problem.lattices):
            rank, rem0, bary32 = simplex(image, self.sig[k])
            if not np.array_equal(bary32, L.bary):
                raise AssertionError("the restated simplex does not reproduce lattice %d's barycentric weights" % k)
            self.raw.append(_raw_features(image, L.d))
            self.rank.append(rank)
            self.rem0.append(rem0)

    def features32(self, k):
        """The build's float32 features at theta0."""
        return (self.raw[k].astype(np.float32) / np.asarray(self.sig[k], np.float32)).astype(np.float32)

    def features(self, k, theta):
        sig = theta[5:7] if k == 0 else theta[0:5]
        return self.raw[k] / np.asarray(sig, np.float64)

    def bary(self, k, theta):
        """float64 barycentric weights at `theta` on the held simplices."""
        d = self.problem.lattices[k].d
        el = _elevate(self.features(k, theta), _scales(d, np.float64))
        v = (el - self.rem0[k]) / (d + 1)
        rows = np.arange(el.shape[0])[:, None]
        rho = np.empty_like(self.rank[k])                 # rho[:, r] = the coordinate of rank d - r
        rho[rows, d - self.rank[k]] = np.arange(d + 1)[None, :]
        vr = v[rows, rho]
        b = vr - np.roll(vr, 1, axis=1)
        b[:, 0] += 1.0
        return b

    def frozen_problem(self, theta):
        """A copy of the problem whose lattices carry the float64 weights at `theta` (norms recomputed)."""
        P = copy.copy(self.problem)
        P._norms = {}
        P.lattices = []
        for k, L in enumerate(self.problem.lattices):
            L2 = copy.copy(L)
            L2.bary = self.bary(k, theta)
            P.lattices.append(L2)
        return P


def _mus(problem, mus):
    """Per lattice (spatial, bilateral) the float64 compatibility {mu_bi, mu_sp} as given, or None (Potts)."""
    if mus is not None:
        return [np.asarray(mus[1], np.float64), np.asarray(mus[0], np.float64)]
    return [None, None]


def forward(P, unary, T, mus=None):
    """Q_0..Q_T in float64 on problem P (Potts weights from its lattices, or mus = (mu_bi, mu_sp))."""
    if mus is None:
        return P.run(unary, T)
    return crf_compat_oracle.run(P, unary, mus, T)


def loss(P, unary, G, T, mus=None):
    return float((forward(P, unary, T, mus)[-1] * G).sum())


def _rot(L, s, rank, mutant=None, magnitude=False):
    """dL/d(features) (N, d) from s (N, d+1) = the per-vertex derivative of a bilinear form w.r.t. the pixel's
    barycentric weights (alpha included): the rank rotation and the transposed elevation (permutohedral.cpp:664-694).
    `magnitude`: the same sums over absolute values (the scale of their float32 rounding before any cancellation)."""
    d = L.d
    rows = np.arange(s.shape[0])[:, None]
    r0 = d - rank
    r1 = (r0 + (2 if mutant == "rank_off_by_one" else 1)) % (d + 1)
    if magnitude:
        gel = (np.abs(s[rows, r0]) + np.abs(s[rows, r1])) / (d + 1)
    else:
        gel = (s[rows, r0] - s[rows, r1]) / s.dtype.type(d + 1)
    sc = _scales(d, s.dtype.type)
    df = np.empty((s.shape[0], d), s.dtype)
    sm = gel[:, 0].copy()
    for j in range(1, d + 1):
        df[:, j - 1] = sc[j - 1] * (sm + j * gel[:, j] if magnitude else sm - s.dtype.type(j) * gel[:, j])
        sm += gel[:, j]
    return df


def theta_grad(frozen, theta, unary, grad_q, T, mus=None, convention="exact", mutant=None, dtype=np.float64,
               splat_order=None, arith="oracle", exp_seed=0):
    """dL/dtheta (7,) in dsrg_crf_params order and dL/dp (7,) in the same order, for L = <grad_q, Q_T>, on the frozen
    lattices at `theta`; plus A (7,): the sum over the pixels of |f_i| times the magnitude of (dL/df)_i's terms before
    they cancel (the scale of a float32 evaluation's rounding error).

    float64: the truth.  float32 (at theta0, on the build's own float32 weights): a model of the device's rounding,
    every array float32 -- the iterates from meanfield64's / crf_compat_oracle's float32 forward (``splat_order``,
    ``arith``, ``exp_seed`` as there), the splats in ``splat_order``, features, blurs, slices and the rotation."""
    f64 = dtype == np.float64
    P = frozen.frozen_problem(theta) if f64 else frozen.problem
    M = grad_q.shape[-1]
    if mus is None:
        Qs = P.run(unary, T, dtype, splat_order, arith, exp_seed=exp_seed)
    else:
        Qs = crf_compat_oracle.run(P, unary, mus, T, dtype, splat_order, arith, exp_seed)
    Qs = [q.reshape(P.N, M).astype(dtype) for q in Qs]
    G = np.asarray(grad_q, np.float64).reshape(P.N, M).astype(dtype)
    norms = P.norms(dtype, None if f64 else splat_order)
    mu = _mus(P, mus)
    for k, L in enumerate(P.lattices):
        mu[k] = (-L.w * np.eye(M) if mu[k] is None else mu[k]).astype(dtype)
    fwd, rev = (L_blur_fwd, L_blur_rev) if convention == "exact" else (L_blur_rev, L_blur_fwd)
    if mutant == "forward_order":
        fwd = rev = L_blur_fwd
    half = dtype(0.5)

    def vjp(q, gt):
        return q * (gt - (gt * q).sum(1)[:, None])

    S = [L.splat_matrix(L.bary, dtype, None if f64 else splat_order) for L in P.lattices]
    alpha = [L.alpha(dtype) for L in P.lattices]
    df = [np.zeros((P.N, L.d), dtype) for L in P.lattices]
    mag = [np.zeros((P.N, L.d)) for L in P.lattices]
    csum = [np.zeros(P.N, dtype) for _ in P.lattices]
    g = vjp(Qs[T], G)
    for t in range(T - 1, -1, -1):
        Gt = np.zeros((P.N, M), dtype)
        for k, L in enumerate(P.lattices):
            n = norms[k][:, None]
            x = -(g @ mu[k])
            y = Qs[t]
            vy_true = L.blur(S[k] @ (n * y), False)
            vx_true = crf_grad_oracle.blur_t(L, S[k] @ (n * x))
            vy, vx = fwd(L, S[k] @ (n * y)), rev(L, S[k] @ (n * x))
            s = ((n * x)[:, None, :] * vy[L.offset]).sum(2) + ((n * y)[:, None, :] * vx[L.offset]).sum(2)
            df[k] += alpha[k] * _rot(L, s, frozen.rank[k], mutant)
            mag[k] += float(alpha[k]) * _rot(L, s.astype(np.float64), frozen.rank[k], magnitude=True)
            kny, ktnx = L.slice(vy_true, False), L.slice(vx_true, False)
            csum[k] += half * norms[k] ** 3 * (x * kny + ktnx * y).sum(1)
            Sk = L.slice(crf_grad_oracle.blur_t(L, S[k] @ (n * g)), False) * n
            Gt -= Sk @ mu[k]
        g = vjp(Qs[t], Gt)
    dp, ab = np.zeros(7), np.zeros(7)
    for k, L in enumerate(P.lattices):
        if T > 0 and mutant != "no_norm":
            v1 = fwd(L, S[k] @ np.ones((P.N, 1), dtype))[:, 0]
            vc = rev(L, S[k] @ csum[k][:, None])[:, 0]
            s = csum[k][:, None] * v1[L.offset] + vc[L.offset]
            df[k] -= alpha[k] * _rot(L, s, frozen.rank[k], mutant)
            mag[k] += float(alpha[k]) * _rot(L, s.astype(np.float64), frozen.rank[k], magnitude=True)
        f = frozen.features(k, theta) if f64 else frozen.features32(k)
        at = slice(5, 7) if k == 0 else slice(0, 5)
        dp[at] = (f * df[k]).sum(0, dtype=dtype)
        ab[at] = (np.abs(f.astype(np.float64)) * mag[k]).sum(0)
    return -dp / theta, dp, ab


def L_blur_fwd(L, v):
    return L.blur(v, False)


def L_blur_rev(L, v):
    return crf_grad_oracle.blur_t(L, v)


def finite_diff(frozen, theta, unary, grad_q, T, mus=None, rel=1e-5):
    """Central differences of <grad_q, Q_T> on the frozen lattices, one sigma at a time."""
    G = np.asarray(grad_q, np.float64)
    out = np.zeros(7)
    for i in range(7):
        h = rel * theta[i]
        tp, tm = theta.copy(), theta.copy()
        tp[i] += h
        tm[i] -= h
        out[i] = (loss(frozen.frozen_problem(tp), unary, G, T, mus)
                  - loss(frozen.frozen_problem(tm), unary, G, T, mus)) / (2 * h)
    return out
