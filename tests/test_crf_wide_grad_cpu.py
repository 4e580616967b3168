"""The CRF gradient above 32 labels without a GPU: the float64 restatements (oracle/crf_grad_oracle,
oracle/crf_compat_oracle) against central differences at 33 and 81 labels and against the reference's own
DenseCRF::gradient (frozen in tests/golden/crf_wide_grad_ref.npz); three wrong backwards outside the bars of the GPU
file's cases; nn.dense_crf_wide's refusals that need no device."""
import os

import numpy as np
import pytest

import helpers
from crf_compat_cases import CompatTruth, compat_mats
from crf_grad_cases import GradTruth, grad_params, upstream
from crf_wide_grad_cases import GOLDEN, GOLDEN_CASES, golden_inputs
from oracle import crf_compat_oracle, crf_grad_oracle, meanfield64

GOLDEN_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", GOLDEN)


def _case(H, W, img, M, sf, T, seed):
    image = helpers.small_image(np.random.RandomState(seed), H, W, img)
    unary = helpers.log_unary(1, H, W, M, seed, scale=1.0)[0]
    p = grad_params(sf, T)
    return meanfield64.Problem(image, p), image, unary, upstream(H, W, M, seed), p


def _indices(rng, shape, n):
    return [tuple(rng.randint(s) for s in shape) for _ in range(n)]


@pytest.mark.parametrize("M", [33, 81])
def test_potts_restatement_meets_finite_differences(M):
    """L = <G, Q_T>: central differences of the float64 forward in a few unaries and in both weights."""
    T = 3
    P, image, unary, G, p = _case(7, 9, "noise", M, 1.0, T, 5)
    gU, gw, _ = crf_grad_oracle.backward(P, P.run(unary, T), G)
    for i in _indices(np.random.RandomState(M), unary.shape, 4):   # the forward takes float32 unaries
        up, um = unary.copy(), unary.copy()
        up[i] += np.float32(1e-2)
        um[i] -= np.float32(1e-2)
        fd = float(((P.run(up, T)[-1] - P.run(um, T)[-1]) * G).sum()) / (float(up[i]) - float(um[i]))
        assert abs(fd - gU[i]) <= 1e-4 * np.abs(gU).max() + 1e-9, (i, fd, gU[i])
    for k, name in enumerate(("w1", "w2")):   # the weights are float32 too: the step is what they hold
        ls, ws = [], []
        for d in (1e-2, -1e-2):
            q = grad_params(p, T)
            setattr(q, name, getattr(p, name) + d)
            ws.append(float(getattr(q, name)))
            ls.append(float((meanfield64.Problem(image, q).run(unary, T)[-1] * G).sum()))
        fd = (ls[0] - ls[1]) / (ws[0] - ws[1])
        assert abs(fd - gw[k]) <= 1e-4 * max(1.0, abs(gw[k])), (name, fd, gw[k])


@pytest.mark.parametrize("M", [33, 81])
def test_matrix_restatement_meets_finite_differences(M):
    """The same for non-symmetric matrices: a few unaries and entries of both matrices in both orders."""
    T = 2
    P, _, unary, G, _ = _case(7, 9, "noise", M, 1.0, T, 6)
    mus = [m.astype(np.float64) for m in compat_mats("nonsym", M, 8)]
    gU, gmu, _ = crf_compat_oracle.backward(P, crf_compat_oracle.run(P, unary, mus, T), G, mus)

    def loss(u, m):
        return float((crf_compat_oracle.run(P, u, m, T)[-1] * G).sum())

    rng = np.random.RandomState(M)
    for i in _indices(rng, unary.shape, 3):
        up, um = unary.copy(), unary.copy()
        up[i] += np.float32(1e-2)
        um[i] -= np.float32(1e-2)
        fd = (loss(up, mus) - loss(um, mus)) / (float(up[i]) - float(um[i]))
        assert abs(fd - gU[i]) <= 1e-4 * np.abs(gU).max() + 1e-9, (i, fd, gU[i])
    eps = 1e-5
    for k in (0, 1):
        l, l2 = rng.randint(M), rng.randint(M)
        for a, b in ((l, l2), (l2, l), (l, l)):
            mp = [m.copy() for m in mus]
            mm = [m.copy() for m in mus]
            mp[k][a, b] += eps
            mm[k][a, b] -= eps
            fd = (loss(unary, mp) - loss(unary, mm)) / (2 * eps)
            assert abs(fd - gmu[k][a, b]) <= 1e-6 * np.abs(gmu[k]).max() + 1e-9, (k, a, b, fd, gmu[k][a, b])


@pytest.mark.parametrize("name", sorted(GOLDEN_CASES))
def test_restatements_reproduce_the_reference(name):
    """The reference's float32 gradient lies within the float32 models' bar of the float64 truth.  Where oracle/_ref is
    built its live result must equal the frozen one."""
    image, unary, G, p, mus = golden_inputs(name)
    P = meanfield64.Problem(image, p)
    with np.load(GOLDEN_PATH) as z:
        frozen = {k.split("/", 1)[1]: z[k] for k in z.files if k.startswith(name + "/")}
    if mus is None:
        if crf_grad_oracle.ref_available():
            gU, gw = crf_grad_oracle.ref_crf_gradient(image, unary, p, G)
            np.testing.assert_array_equal(gU, frozen["grad_unary"])
            np.testing.assert_array_equal(np.array(gw, np.float32), frozen["grad_w"])
        truth = GradTruth(P, unary, G, p.n_iters)
        truth.check(frozen["grad_unary"], frozen["grad_w"], "reference %s:" % name)
        assert np.abs(truth.gU).max() > 1e-3
        return
    if crf_compat_oracle.ref_available():
        q, gU, lg = crf_compat_oracle.ref_crf_compat(image, unary, p, mus[0], mus[1], G)
        np.testing.assert_array_equal(q, frozen["q"])
        np.testing.assert_array_equal(gU, frozen["grad_unary"])
        np.testing.assert_array_equal(lg["sp"], frozen["lbl_cmp_grad_sp"])
    truth = CompatTruth(P, unary, G, p.n_iters, mus)
    truth.check(frozen["q"], frozen["grad_unary"], None, "reference %s:" % name)
    for k, i in (("bi", 0), ("sp", 1)):
        want = crf_compat_oracle.pack(truth.gmu[i])
        bar = crf_compat_oracle.pack(truth.bar_mu[i])
        got = frozen["lbl_cmp_grad_" + k]
        assert (np.abs(got - want) <= bar).all(), (k, np.abs(got - want).max())


def _backward_without_dot(problem, Qs, G):
    """crf_grad_oracle.backward's float32 oracle arithmetic with the <G, Q> term of the soft-max VJP dropped."""
    P = problem
    M = G.shape[-1]
    T = len(Qs) - 1
    Q = [np.asarray(q, np.float32).reshape(P.N, M) for q in Qs]
    norms = P.norms(np.float32)
    S = [L.splat_matrix(L.bary, np.float32, None) for L in P.lattices]
    g = Q[T] * G.reshape(P.N, M).astype(np.float32)
    gU = g.copy()
    for t in range(T - 1, -1, -1):
        Gt = np.zeros((P.N, M), np.float32)
        for k, (L, n) in enumerate(zip(P.lattices, norms)):
            v = crf_grad_oracle.blur_t(L, S[k] @ (g * n[:, None]).astype(np.float32))
            Gt = Gt + np.float32(L.w) * (L.slice(v, False) * n[:, None])
        g = Q[t] * Gt
        gU = gU + g
    return gU.reshape(P.H, P.W, M)


@pytest.mark.parametrize("M", [33, 81])
def test_mutants_fall_outside_the_bars(M):
    """The wide GPU file's cases must catch each wrong backward: the blur of K^T over axes 0..d, mu where mu^T belongs,
    and the soft-max VJP without its <G, Q> term -- on a 23 x 27 photo, 3 iterations (test_wide_grad_on_every_image_kind's
    shape)."""
    T = 3
    P, _, unary, G, _ = _case(23, 27, "photo", M, 1.0, T, 11)
    truth = GradTruth(P, unary, G, T, mutant="transpose_forward_order")
    q32 = P.run(unary, T, np.float32)
    assert float(np.abs(truth.mutant[0] - truth.gU).max()) > 10 * truth.bar_u
    assert float(np.abs(_backward_without_dot(P, q32, G) - truth.gU).max()) > 10 * truth.bar_u
    mus = compat_mats("nonsym", M, 2)
    ct = CompatTruth(P, unary, G, T, mus, mutants=("mu_untransposed",))
    over = ct.over(*ct.mutants["mu_untransposed"])
    assert max(over) > 10, over


def test_dense_crf_wide_refusals_without_a_gpu():
    torch = pytest.importorskip("torch")
    from dsrg_b200 import nn
    u = torch.zeros((2, 40, 5, 6))
    im = torch.zeros((2, 5, 6, 3), dtype=torch.uint8)
    for bad in (torch.zeros((2, 256, 5, 6)), torch.zeros((2, 40, 5)), torch.zeros((2, 40, 5, 6), dtype=torch.int32)):
        with pytest.raises(ValueError):
            nn.dense_crf_wide(bad, im)
    with pytest.raises(ValueError, match="image"):
        nn.dense_crf_wide(u, im[:1])
    with pytest.raises(ValueError, match="CUDA"):
        nn.dense_crf_wide(u, im)
    with pytest.raises(ValueError, match="at most 32 labels"):
        nn.dense_crf(u, im)
