"""oracle/crf_grad_oracle.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The checkers of the CRF gradient (DenseCRF::gradient, densecrf.cpp:238-297):

* ``ref_crf_gradient`` -- the reference's own gradient, built by oracle/grad.mk into _ref/libdensecrf_grad_ref.so
  (when the reference is present; the built .so travels with the tree)
* ``backward`` -- the same backward restated in numpy on a meanfield64.Problem's lattices (the oracle's, which the
  engine reproduces exactly), in float64 and in the float32 models meanfield64's forward offers:

      g_T = Q_T (G - <G, Q_T>);  for t = T-1..0: S_k = F_k^T(g_{t+1}), dL/dw_k += <S_k, Q_t>,
      g_t = Q_t (G_t - <G_t, Q_t>) with G_t = sum_k w_k S_k;   dL/dU = sum_t g_t

  F^T = norm K^T (norm .) with alpha: the forward's splat and slice around K^T, the blur over axes d..0
  (permutohedral.cpp:556 with reverse).

Only tests/ may import this module.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from . import crf_oracle

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_ref", "libdensecrf_grad_ref.so")
_REF = None

# name -> what the float32 backward then does wrong
MUTANTS = {"transpose_forward_order": "the transposed blur K^T taken over axes 0..d (K's order) instead of d..0"}


def build(force=False):
    if os.path.exists("/root/reference/CRF/src/densecrf.cpp") and (force or not os.path.exists(_SO)):
        subprocess.check_call(["make", "-C", _HERE, "-f", "grad.mk", "ref"], stdout=subprocess.DEVNULL)


def ref_available():
    return os.path.exists(_SO)


def _ref():
    global _REF
    if _REF is None:
        R = C.CDLL(_SO)
        f32p, u8p = crf_oracle._f32p, crf_oracle._u8p
        R.ref_densecrf_gradient.argtypes = ([C.c_int] * 3 + [f32p] + [C.c_float] * 9 + [u8p, C.c_int, f32p, f32p, f32p])
        _REF = R
    return _REF


def ref_crf_gradient(image, unary, params, grad_q):
    """The reference's DenseCRF::gradient for the CRF DenseCRFWrapper builds with `params` (a dsrg_crf_params:
    weights, sigmas, n_iters): image (H, W, 3) uint8, unary (H, W, M) the values CRF() takes (energy = -unary),
    grad_q (H, W, M) = dL/dQ_T.  -> (dL/dunary (H, W, M), (dL/dw1, dL/dw2)) in float32: the reference's unary_grad
    (taken w.r.t. the energy) negated, its lbl_cmp_grad ({w2, w1}: the Gaussian term is added first) reordered."""
    H, W, M = unary.shape
    ug = np.empty(H * W * M, np.float32)
    lg = np.empty(2, np.float32)
    p = params
    _ref().ref_densecrf_gradient(W, H, M, np.ascontiguousarray(-unary.ravel(), np.float32), p.w1, p.theta_alpha_x,
                                 p.theta_alpha_y, p.theta_beta_r, p.theta_beta_g, p.theta_beta_b, p.w2,
                                 p.theta_gamma_x, p.theta_gamma_y, np.ascontiguousarray(image, np.uint8).ravel(),
                                 int(p.n_iters), np.ascontiguousarray(grad_q, np.float32).ravel(), ug, lg)
    return -ug.reshape(H, W, M), (float(lg[1]), float(lg[0]))


def blur_t(L, v, mutant=None):
    """K^T of one meanfield64.Lattice: the axis blurs d..0 (0..d under the mutant), o + 0.5 (n1 + n2) each."""
    axes = range(L.d + 1) if mutant == "transpose_forward_order" else range(L.d, -1, -1)
    half = v.dtype.type(0.5)
    for j in axes:
        new = np.empty_like(v)
        new[0] = 0
        new[1:] = v[1:] + half * (v[L.n1[j]] + v[L.n2[j]])
        v = new
    return v


def backward(problem, Qs, grad_q, dtype=np.float64, splat_order=None, arith="oracle", mutant=None):
    """dL/dU and the Potts gradients through the iterates ``Qs`` = problem.run(...) (Q_0..Q_T) for dL/dQ_T = grad_q
    (H, W, M).  -> (dL/dU (H, W, M), (dL/dw1, dL/dw2), (A1, A2)) with A_k the sum of |S_k|·|Q_t| over the terms of
    w_k's gradient (the scale of a float32 sum's rounding error).  float32: ``arith="oracle"`` is the oracle's
    splat (in ``splat_order``) and slice, ``arith="device"`` k_mf_tile_bwd's operation order (wn = bary·norm, the
    slice an fma chain from zero with weights alpha·wn, the dot products and G_t as fma chains)."""
    P = problem
    M = grad_q.shape[-1]
    T = len(Qs) - 1
    Q = [np.asarray(q).reshape(P.N, M).astype(dtype) for q in Qs]
    G = np.asarray(grad_q, np.float64).reshape(P.N, M).astype(dtype)
    norms = P.norms(dtype, splat_order)
    device = arith == "device"
    f64 = np.float64

    def fma(a, b, c):
        return (a.astype(f64) * b + c).astype(dtype) if device else a * b + c

    def vjp(q, gt):
        if device:
            dot = np.zeros(P.N, dtype)
            for k in range(M):
                dot = fma(gt[:, k], q[:, k], dot)
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
    gw, ga = [0.0, 0.0], [0.0, 0.0]      # lattice order: spatial (w2), bilateral (w1)
    for t in range(T - 1, -1, -1):
        Gt = np.zeros((P.N, M), dtype)
        for k, (L, n) in enumerate(zip(P.lattices, norms)):
            if device:
                v = blur_t(L, S[k] @ g, mutant)
                wr = (L.alpha(np.float32) * wn[k]).astype(np.float32)
                s = np.zeros((P.N, M), dtype)
                for r in range(L.d + 1):
                    s = fma(wr[:, r, None], v[L.offset[:, r]], s)
                Gt = fma(np.full((P.N, M), L.w, dtype), s, Gt) if k else (dtype(L.w) * s).astype(dtype)
            else:
                v = blur_t(L, S[k] @ (g * n[:, None]).astype(dtype), mutant)
                s = L.slice(v, False) * n[:, None]
                Gt = Gt + dtype(L.w) * s
            prod = s.astype(f64) * Q[t]
            gw[k] += float(prod.sum())
            ga[k] += float(np.abs(prod).sum())
        g = vjp(Q[t], Gt)
        gU = gU + g
    return gU.reshape(P.H, P.W, M), (gw[1], gw[0]), (ga[1], ga[0])
