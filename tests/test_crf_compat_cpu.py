"""The compatibility-matrix CRF's float64 restatement (oracle/crf_compat_oracle) against the Potts restatements it
generalises, against the reference's own MatrixCompatibility inference and gradient, and against central finite
differences; its float32 models against their bar, and the bar against three wrong backwards.  No GPU."""
import os

import numpy as np
import pytest

import helpers
from crf_compat_cases import (COMPAT_ITERS, COMPAT_M, GOLDEN, GOLDEN_CASES, CompatTruth, compat_mats,
                              golden_inputs)
from crf_grad_cases import grad_params, upstream
from oracle import crf_compat_oracle, crf_grad_oracle, meanfield64

GOLDEN_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", GOLDEN)


def _case(H, W, img, M, sf, T, seed):
    image = helpers.small_image(np.random.RandomState(seed), H, W, img)
    unary = helpers.log_unary(1, H, W, M, seed, scale=1.0)[0]
    p = grad_params(sf, T)
    return meanfield64.Problem(image, p), image, unary, upstream(H, W, M, seed), p


@pytest.mark.parametrize("T", [1, 3])
def test_potts_matrices_equal_the_potts_restatements(T):
    """mu = -w I: the forward is meanfield64's, dL/dU crf_grad_oracle's, and -trace(dL/dmu_k) its dL/dw_k."""
    P, _, unary, G, p = _case(9, 11, "noise", 5, 1.0, T, 4)
    mus = compat_mats("potts", 5, 0, p.w1, p.w2)
    q = crf_compat_oracle.run(P, unary, mus, T)
    q0 = P.run(unary, T)
    for a, b in zip(q, q0):
        np.testing.assert_allclose(a, b, rtol=0, atol=1e-12)
    gU, gmu, _ = crf_compat_oracle.backward(P, q, G, mus)
    gU0, gw0, _ = crf_grad_oracle.backward(P, q0, G)
    np.testing.assert_allclose(gU, gU0, rtol=0, atol=1e-12)
    for i in (0, 1):
        assert abs(-np.trace(gmu[i]) - gw0[i]) <= 1e-12 * max(1.0, abs(gw0[i])), (i, -np.trace(gmu[i]), gw0[i])


@pytest.mark.parametrize("name", sorted(GOLDEN_CASES))
def test_float64_matches_the_reference_matrix_compatibility(name):
    """The reference (float32, symmetric mu) lies within the float32 models' bar of the float64 truth: marginals,
    dL/dunary, and its packed lbl_cmp_grad against the truth folded as g(i,j) + g(j,i).  Where oracle/_ref is built
    its live result must equal the frozen one."""
    image, unary, G, p, mus = golden_inputs(name)
    truth = CompatTruth(meanfield64.Problem(image, p), unary, G, p.n_iters, mus)
    with np.load(GOLDEN_PATH) as z:
        q, gU = z[name + "/q"], z[name + "/grad_unary"]
        lg = {"sp": z[name + "/lbl_cmp_grad_sp"], "bi": z[name + "/lbl_cmp_grad_bi"]}
    if crf_compat_oracle.ref_available():
        lq, lu, llg = crf_compat_oracle.ref_crf_compat(image, unary, p, mus[0], mus[1], G)
        np.testing.assert_array_equal(lq, q)
        np.testing.assert_array_equal(lu, gU)
        for k in ("sp", "bi"):
            np.testing.assert_array_equal(llg[k], lg[k])
    truth.check(q, gU, None, "reference %s:" % name)
    for k, i in (("bi", 0), ("sp", 1)):
        want = crf_compat_oracle.pack(truth.gmu[i])
        bar = crf_compat_oracle.pack(truth.bar_mu[i])
        assert (np.abs(lg[k] - want) <= bar).all(), (k, np.abs(lg[k] - want).max(), bar.min())
    assert np.abs(truth.gU).max() > 1e-3 and np.abs(truth.gmu).max() > 1e-3


@pytest.mark.parametrize("kind", ["nonsym", "sym"])
def test_float64_gradient_matches_finite_differences(kind):
    """L = <G, Q_T>: central differences of the float64 forward in a few unaries and in entries of both matrices,
    off the diagonal in both orders (a non-symmetric mu tells mu from mu^T)."""
    T, M = 3, 4
    P, _, unary, G, p = _case(7, 9, "noise", M, 1.0, T, 3)
    mus = [m.astype(np.float64) for m in compat_mats(kind, M, 8)]
    gU, gmu, _ = crf_compat_oracle.backward(P, crf_compat_oracle.run(P, unary, mus, T), G, mus)

    def loss(u, m):
        return float((crf_compat_oracle.run(P, u, m, T)[-1] * G).sum())

    rng = np.random.RandomState(1)
    for _ in range(3):
        i = tuple(rng.randint(s) for s in unary.shape)
        up, um = unary.copy(), unary.copy()
        up[i] += np.float32(1e-2)
        um[i] -= np.float32(1e-2)
        fd = (loss(up, mus) - loss(um, mus)) / (float(up[i]) - float(um[i]))
        assert abs(fd - gU[i]) <= 1e-4 * np.abs(gU).max() + 1e-9, (i, fd, gU[i])
    h = 1e-5
    for k in (0, 1):
        for (l, l2) in ((0, 0), (1, 2), (2, 1), (3, 0)):
            mp = [m.copy() for m in mus]
            mm = [m.copy() for m in mus]
            mp[k][l, l2] += h
            mm[k][l, l2] -= h
            fd = (loss(unary, mp) - loss(unary, mm)) / (2 * h)
            assert abs(fd - gmu[k, l, l2]) <= 1e-6 * np.abs(gmu[k]).max() + 1e-9, (k, l, l2, fd, gmu[k, l, l2])


CPU_CASES = ([("smooth", M, 3, "nonsym") for M in COMPAT_M] + [("noise", 21, T, "nonsym") for T in COMPAT_ITERS]
             + [("smooth", 6, 2, kind) for kind in ("zero", "potts", "sym", "diag", "classic")])


@pytest.mark.parametrize("img,M,T,kind", CPU_CASES)
def test_float32_models_lie_within_the_bar_and_the_mutants_beyond(img, M, T, kind):
    H, W = helpers.FUSED_SHAPES[img]
    H, W = H // 2, W // 2
    P, _, unary, G, p = _case(H, W, img, M, 1.0, T, 11 + M)
    mus = compat_mats(kind, M, 13 + M)
    # with two labels g_t and S are multiples of (1, -1), and (mu - mu^T) S then lies along (1, 1), which the softmax
    # VJP removes: mu and mu^T give the same dL/dU there, so the mutants are checked from three labels on
    mutants = list(crf_compat_oracle.MUTANTS) if kind == "nonsym" and T > 0 and M > 2 else []
    truth = CompatTruth(P, unary, G, T, mus, mutants=mutants)
    for k, (q, u, g) in enumerate(truth.models):
        truth.check(q, u, g, "model %d:" % k)
    if M > 1:   # the bar is float32 noise, well below the gradient itself
        assert truth.bar_u <= 2e-2 * truth.scale, (truth.bar_u, truth.scale)
    if T == 0:
        assert not truth.gmu.any()
    for name, (u, g) in truth.mutants.items():
        assert max(truth.over(u, g)) > 1.0, "mutant %s stays within the bar" % name


@pytest.mark.parametrize("H,W,img", helpers.MF64_TINY)
def test_phantom_lane_shapes(H, W, img):
    P, image, unary, G, p = _case(H, W, img, helpers.MF64_TINY_M, 1.0, 3, helpers.MF64_TINY_SEED)
    mus = compat_mats("sym", helpers.MF64_TINY_M, 2)
    truth = CompatTruth(P, unary, G, 3, mus)
    for q, u, g in truth.models:
        truth.check(q, u, g)
    if crf_compat_oracle.ref_available():
        q, u, lg = crf_compat_oracle.ref_crf_compat(image, unary, p, mus[0], mus[1], G)
        truth.check(q, u, None, "reference:")
