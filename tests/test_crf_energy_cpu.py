"""The CRF energy's float64 restatement (oracle/crf_energy_oracle.py) without a GPU: against the reference's own
klDivergence frozen in tests/golden/crf_energy_ref.npz, its gradient against central finite differences, and the
refusals of nn.dense_crf_energy and the C symbols that need no device."""
import os
import re

import numpy as np
import pytest

import helpers
from crf_compat_cases import compat_mats
from crf_energy_cases import GOLDEN, GOLDEN_CASES, golden_inputs, grad_terms, library_mus, problem, q_of
from crf_fgrad_cases import features_of
from crf_grad_cases import grad_params
from dsrg_b200 import _lib
from oracle import crf_energy_oracle as E

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# The reference sums each pairwise term in float32, sequentially over the N * M products (Eigen's sum, oracle/
# eigen_shim), after a float32 filter: on these 99-pixel images that is a few 2^-24 relative per value and about
# sqrt(N M) of them in the sum.  The restatement is float64, so the difference is that float32 rounding: 2^-18 of the
# magnitude sum (the largest measured was 2.4e-7 of it, below 2^-21).
GOLDEN_REL = 2.0 ** -18


@pytest.mark.parametrize("name", sorted(GOLDEN_CASES))
def test_restatement_reproduces_the_reference_kl_divergence(name):
    q, unary, p, m, image, feats = golden_inputs(name)
    want = np.load(os.path.join(ROOT, "tests", "golden", GOLDEN))[name + "/terms"]
    got, scale = E.terms(problem(image, p, feats), q, unary, library_mus(m))
    assert np.all(np.abs(got - want) <= GOLDEN_REL * scale + 1e-12), (got, want, scale)
    if unary is None:
        assert got[1] == 0.0 and want[1] == 0.0


def _tiny(mu, bil, M=3, seed=0):
    H, W = 5, 6
    image = helpers.small_image(np.random.RandomState(40 + seed), H, W, "noise")
    p = grad_params(1.0, 0)
    feats = None if bil == "image" else features_of(bil, image, p, seed)
    rng = np.random.RandomState(60 + seed)
    q = rng.uniform(0.05, 1.2, (H, W, M))             # away from the clamp, so that the energy is smooth there
    unary = rng.randn(H, W, M)
    return problem(image, p, feats), q, unary, (compat_mats(mu, M, 5) if mu else None)


def _fd(P, q, unary, g, mus, d, h, of_unary=False):
    if of_unary:
        return (E.energy_of(P, q, unary + h * d, g, mus) - E.energy_of(P, q, unary - h * d, g, mus)) / (2 * h)
    return (E.energy_of(P, q + h * d, unary, g, mus) - E.energy_of(P, q - h * d, unary, g, mus)) / (2 * h)


@pytest.mark.parametrize("bil", ["image", "random"])
@pytest.mark.parametrize("mu", [None, "nonsym"])
def test_gradient_matches_finite_differences(mu, bil):
    P, q, unary, mus = _tiny(mu, bil)
    g = grad_terms(1, 3)[0].astype(np.float64)
    dq, du, _ = E.gradient(P, q, unary, g, mus)
    rng = np.random.RandomState(9)
    for _ in range(2):   # random directions: every pixel and label at once
        d = rng.randn(*q.shape)
        for of_unary, want in ((False, dq), (True, du)):
            fd = _fd(P, q, unary, g, mus, d, 1e-6, of_unary)
            assert abs(fd - (want * d).sum()) <= 1e-6 * max(1.0, abs(fd)), (of_unary, fd, (want * d).sum())
    for pix in ((0, 0, 0), (2, 3, 1), (4, 5, 2)):   # single entries, the last pixel included
        d = np.zeros_like(q)
        d[pix] = 1.0
        fd = _fd(P, q, unary, g, mus, d, 1e-6)
        assert abs(fd - dq[pix]) <= 1e-6 * max(1.0, abs(fd)), (pix, fd, dq[pix])


def test_symmetrised_transpose_is_not_the_gradient():
    """mu F + mu^T F^T differs from 2 mu F wherever a blur neighbour is missing: the finite differences tell them
    apart, so the device's gradient must take the transposed blur (as the restatement does)."""
    P, q, unary, mus = _tiny("nonsym", "image")
    g = np.array([0.0, 0.0, 1.0, 1.0])
    dq, _, _ = E.gradient(P, q, unary, g, mus)
    sym = np.zeros_like(dq).reshape(P.N, -1)
    Q = q.reshape(P.N, -1)
    for k, mu in enumerate(E._mus(P, mus, q.shape[-1])):
        F = E.filt(P, k, Q)
        Ft_as_F = F.copy()
        sym += F @ mu.T + Ft_as_F @ mu
    d = np.random.RandomState(4).randn(*q.shape)
    fd = _fd(P, q, unary, g, mus, d, 1e-6)
    exact, wrong = abs(fd - (dq * d).sum()), abs(fd - (sym.reshape(q.shape) * d).sum())
    assert exact <= 1e-6 * abs(fd) and wrong > 1e3 * exact + 1e-6 * abs(fd), (exact, wrong, fd)


def test_entropy_derivative_at_and_below_the_clamp():
    """Q log max(Q, 1e-20f): at Q = 0 and at Q = 1e-25 the derivative is log 1e-20f, as the formula is written."""
    P, q, unary, mus = _tiny(None, "image")
    q = q.copy()
    q[0, 0, 0], q[1, 1, 1] = 0.0, 1e-25
    g = np.array([1.0, 0.0, 0.0, 0.0])
    dq, _, _ = E.gradient(P, q, None, g, mus)
    ent = lambda x: x * np.log(max(x, E.EPS))   # the pixel's own entropy term: the sum's rounding hides it
    for pix in ((0, 0, 0), (1, 1, 1)):
        assert dq[pix] == np.log(E.EPS)
        fd = (ent(q[pix] + 1e-23) - ent(q[pix] - 1e-23)) / 2e-23
        assert abs(fd - np.log(E.EPS)) <= 1e-9 * abs(fd), (pix, fd)


def test_one_hot_energy_is_the_labelling_energy():
    """A one-hot q has no entropy, and its Potts pairwise terms are -w times the kernel mass between equal labels."""
    P, _, unary, _ = _tiny(None, "image", M=4)
    q = q_of("onehot", 5, 6, 4, 2).astype(np.float64)
    t, _ = E.terms(P, q, unary)
    assert t[0] == 0.0
    Q = q.reshape(P.N, 4)
    for k, L in enumerate(P.lattices):
        same = E.filt(P, k, Q)[np.arange(P.N), Q.argmax(1)].sum()
        assert abs(t[2 + k] - (-L.w * same)) <= 1e-12 * abs(t[2 + k])


def test_new_symbols_are_declared_and_exported():
    header = open(os.path.join(ROOT, "include", "dsrg_b200.h")).read()
    L = _lib.lib()
    for name in ("dsrg_crf_energy_dev", "dsrg_crf_energy_backward_dev"):
        assert re.search(r"\bint %s\(" % name, header), name
        assert name in _lib.SIGNATURES
        getattr(L, name)
    assert L.dsrg_version() >= 118
    assert "crf_energy" in [L.dsrg_profile_tag_name(t).decode() for t in range(L.dsrg_profile_tag_count())]


def test_dense_crf_energy_refusals_without_gpu():
    torch = pytest.importorskip("torch")
    from dsrg_b200 import nn
    q = torch.zeros(1, 3, 4, 5)
    img = torch.zeros(1, 4, 5, 3, dtype=torch.uint8)
    f = torch.zeros(1, 5, 4, 5)
    with pytest.raises(ValueError, match="at most 32 labels"):
        nn.dense_crf_energy(torch.zeros(1, 33, 4, 5), None, torch.zeros(1, 4, 5, 3, dtype=torch.uint8))
    with pytest.raises(ValueError, match="image is not used"):
        nn.dense_crf_energy(q, None, img, features_bi=f)
    with pytest.raises(ValueError, match="image must be"):
        nn.dense_crf_energy(q, None, None)
    with pytest.raises(ValueError, match="unary must have"):
        nn.dense_crf_energy(q, torch.zeros(1, 2, 4, 5), img)
    for kw in (dict(w1=torch.tensor(3.0, requires_grad=True)), dict(compat_bi=torch.zeros(3, 3, requires_grad=True)),
               dict(theta_sp=torch.ones(2, requires_grad=True))):
        with pytest.raises(ValueError, match="requires grad"):
            nn.dense_crf_energy(q, None, img, **kw)
    with pytest.raises(ValueError, match="requires grad"):
        nn.dense_crf_energy(q, None, None, features_bi=f.requires_grad_())
    with pytest.raises(ValueError, match="CUDA tensor"):
        nn.dense_crf_energy(q, None, img)
