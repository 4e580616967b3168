"""oracle/crf_compat_oracle.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The dense CRF with a label-compatibility matrix per kernel (the reference's MatrixCompatibility,
labelcompatibility.cpp:64-108, applied as given) and its gradient:

    forward : t_{t+1} = U - mu_sp F_sp(Q_t) - mu_bi F_bi(Q_t);  Q_{t+1} = softmax(t_{t+1})
    backward: g_T = Q_T (G - <G, Q_T>);  for t = T-1..0: S_k = F_k^T(g_{t+1}),  dL/dmu_k += -S_k^T Q_t,
              g_t = Q_t (G_t - <G_t, Q_t>) with G_t = -sum_k S_k mu_k;   dL/dU = sum_t g_t

restated on a meanfield64.Problem's lattices with crf_grad_oracle's transposed blur, in float64 and in float32 models:
``arith="oracle"`` filters as meanfield64's float32 forward does (``splat_order`` as there) and applies mu as a
float32 matrix product; ``arith="device"`` is meanfield.cu's operation order under MODE_COMPAT (each lattice sliced
from zero by an fma chain with weights alpha·wn, then its mat-vec as an fma chain over the labels in ascending order,
the spatial lattice first).

* ``ref_crf_compat`` -- the reference's own inference and gradient with MatrixCompatibility on both terms, built by
  oracle/compat.mk into _ref/libdensecrf_compat_ref.so (when the reference is present; the .so travels with the tree)

Only tests/ may import this module.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from . import crf_grad_oracle, crf_oracle
from .meanfield64 import EX2_REL

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_ref", "libdensecrf_compat_ref.so")
_REF = None

# name -> what the float32 backward then does wrong
MUTANTS = {
    "mu_untransposed": "G_t = -sum_k S_k mu_k^T (mu instead of mu^T)",
    "outer_transposed": "dL/dmu_k from Q_t (x) S_k instead of S_k (x) Q_t",
    "transpose_forward_order": crf_grad_oracle.MUTANTS["transpose_forward_order"],
}


def build(force=False):
    if os.path.exists("/root/reference/CRF/src/densecrf.cpp") and (force or not os.path.exists(_SO)):
        subprocess.check_call(["make", "-C", _HERE, "-f", "compat.mk", "ref"], stdout=subprocess.DEVNULL)


def ref_available():
    return os.path.exists(_SO)


def _ref():
    global _REF
    if _REF is None:
        R = C.CDLL(_SO)
        f32p, u8p = crf_oracle._f32p, crf_oracle._u8p
        R.ref_densecrf_compat.argtypes = ([C.c_int] * 3 + [f32p, f32p] + [C.c_float] * 5 + [f32p] + [C.c_float] * 2
                                          + [u8p, C.c_int, f32p, f32p, f32p, f32p])
        _REF = R
    return _REF


def ref_crf_compat(image, unary, params, mu_bi, mu_sp, grad_q):
    """The reference CRF of DenseCRFWrapper with MatrixCompatibility(mu_sp), MatrixCompatibility(mu_bi) (it stores and
    applies (m + m^T) / 2) and `params`' sigmas and n_iters: image (H, W, 3) uint8, unary (H, W, M) the values CRF()
    takes, grad_q (H, W, M) = dL/dQ_T.  -> (Q_T (H, W, M), dL/dunary (H, W, M), lbl_cmp_grad: {"sp": ..., "bi": ...}
    each packed M (M + 1) / 2 (upper triangle row-major, g(i,j) + g(j,i) off the diagonal)), float32."""
    H, W, M = unary.shape
    q = np.empty(H * W * M, np.float32)
    ug = np.empty(H * W * M, np.float32)
    P = M * (M + 1) // 2
    lg = np.empty(2 * P, np.float32)
    p = params
    f = lambda m: np.ascontiguousarray(m, np.float32).ravel()
    _ref().ref_densecrf_compat(W, H, M, f(-unary), f(mu_bi), p.theta_alpha_x, p.theta_alpha_y, p.theta_beta_r,
                               p.theta_beta_g, p.theta_beta_b, f(mu_sp), p.theta_gamma_x, p.theta_gamma_y,
                               np.ascontiguousarray(image, np.uint8).ravel(), int(p.n_iters), f(grad_q), q, ug, lg)
    return q.reshape(H, W, M), -ug.reshape(H, W, M), {"sp": lg[:P].copy(), "bi": lg[P:].copy()}


def pack(g):
    """A full (M, M) gradient folded as the reference's MatrixCompatibility::gradient packs it."""
    M = g.shape[0]
    return np.array([g[i, j] + (g[j, i] if i != j else 0.0) for i in range(M) for j in range(i, M)])


def _softmax(t, dtype, device, rng):
    x = t - t.max(1, keepdims=True)
    if device:
        e = (np.exp(x.astype(np.float64)) * (1.0 + rng.uniform(-EX2_REL, EX2_REL, x.shape))).astype(np.float32)
    else:
        e = np.exp(x.astype(np.float64)).astype(dtype)
    s = np.zeros(t.shape[0], dtype)
    for k in range(t.shape[1]):
        s += e[:, k]
    return e * (np.float32(1.0) / s)[:, None] if device else e / s[:, None]


def _device_slice(L, wn, v):
    """meanfield.cu's slice from zero: an fma chain over the incidences with weights alpha·wn."""
    wr = (L.alpha(np.float32) * wn).astype(np.float32)
    s = np.zeros((L.N, v.shape[1]), np.float32)
    for r in range(L.d + 1):
        s = (wr[:, r, None].astype(np.float64) * v[L.offset[:, r]] + s).astype(np.float32)
    return s


def _device_matvec(t, mu, s, transpose):
    """t -= mu s per pixel (t -= mu^T s with `transpose`) as fma chains over the labels l' ascending."""
    for l2 in range(mu.shape[0]):
        col = mu[l2, :] if transpose else mu[:, l2]
        t = ((-col.astype(np.float64))[None, :] * s[:, l2, None] + t).astype(np.float32)
    return t


def run(problem, unary, mus, n_iters, dtype=np.float64, splat_order=None, arith="oracle", exp_seed=0):
    """Q_0..Q_n_iters ((H, W, M) arrays of `dtype`) for unary (H, W, M) and mus = (mu_bi, mu_sp)."""
    P = problem
    M = unary.shape[-1]
    U = np.ascontiguousarray(unary, np.float32).reshape(P.N, M).astype(dtype)
    norms = P.norms(dtype, splat_order)
    device = arith == "device"
    rng = np.random.RandomState(exp_seed)
    mu = [np.asarray(mus[1], np.float64).astype(dtype), np.asarray(mus[0], np.float64).astype(dtype)]   # lattice order
    if device:
        assert dtype == np.float32
        wn = [(L.bary * n[:, None]).astype(np.float32) for L, n in zip(P.lattices, norms)]
        S = [L.splat_matrix(w, dtype, splat_order) for L, w in zip(P.lattices, wn)]
    Q = _softmax(U, dtype, device, rng)
    out = [Q]
    for _ in range(n_iters):
        t = U.copy()
        for k, (L, n) in enumerate(zip(P.lattices, norms)):
            if device:
                t = _device_matvec(t, mu[k], _device_slice(L, wn[k], L.blur(S[k] @ Q, False)), False)
            else:
                f = L.filter(Q * n[:, None], dtype, splat_order) * n[:, None]
                t = t - (f @ mu[k].T).astype(dtype)
        Q = _softmax(t, dtype, device, rng)
        out.append(Q)
    return [q.reshape(P.H, P.W, M) for q in out]


def backward(problem, Qs, grad_q, mus, dtype=np.float64, splat_order=None, arith="oracle", mutant=None):
    """dL/dU and dL/dmu through the iterates Qs = run(...) for dL/dQ_T = grad_q (H, W, M).  -> (dL/dU (H, W, M),
    dL/dmu (2, M, M) {bi, sp}, A (2, M, M)) with A the sum of |S_k|·|Q_t| over each entry's terms (the scale of a
    float32 sum's rounding error)."""
    P = problem
    M = grad_q.shape[-1]
    T = len(Qs) - 1
    Q = [np.asarray(q).reshape(P.N, M).astype(dtype) for q in Qs]
    G = np.asarray(grad_q, np.float64).reshape(P.N, M).astype(dtype)
    norms = P.norms(dtype, splat_order)
    device = arith == "device"
    mu = [np.asarray(mus[1], np.float64).astype(dtype), np.asarray(mus[0], np.float64).astype(dtype)]
    blur_mutant = mutant if mutant == "transpose_forward_order" else None

    def vjp(q, gt):
        if device:
            dot = np.zeros(P.N, dtype)
            for k in range(M):
                dot = (gt[:, k].astype(np.float64) * q[:, k] + dot).astype(dtype)
        else:
            dot = (gt * q).sum(1)
        return q * (gt - dot[:, None])

    if device:
        assert dtype == np.float32
        wn = [(L.bary * n[:, None]).astype(np.float32) for L, n in zip(P.lattices, norms)]
    else:
        wn = [L.bary for L in P.lattices]
    S = [L.splat_matrix(w, dtype, splat_order) for L, w in zip(P.lattices, wn)]
    g = vjp(Q[T], G)
    gU = g.copy()
    gmu = [np.zeros((M, M)), np.zeros((M, M))]     # lattice order: spatial, bilateral
    amu = [np.zeros((M, M)), np.zeros((M, M))]
    for t in range(T - 1, -1, -1):
        Gt = np.zeros((P.N, M), dtype)
        for k, (L, n) in enumerate(zip(P.lattices, norms)):
            if device:
                s = _device_slice(L, wn[k], crf_grad_oracle.blur_t(L, S[k] @ g, blur_mutant))
                Gt = _device_matvec(Gt, mu[k], s, mutant != "mu_untransposed")
            else:
                v = crf_grad_oracle.blur_t(L, S[k] @ (g * n[:, None]).astype(dtype), blur_mutant)
                s = L.slice(v, False) * n[:, None]
                Gt = Gt - (s @ (mu[k].T if mutant == "mu_untransposed" else mu[k])).astype(dtype)
            a, b = (Q[t], s) if mutant == "outer_transposed" else (s, Q[t])
            if dtype == np.float64:
                gmu[k] -= a.T @ b
            else:
                gmu[k] -= (a.T @ b).astype(np.float64)
            amu[k] += np.abs(s.astype(np.float64)).T @ np.abs(Q[t].astype(np.float64))
        g = vjp(Q[t], Gt)
        gU = gU + g
    return gU.reshape(P.H, P.W, M), np.stack([gmu[1], gmu[0]]), np.stack([amu[1], amu[0]])
