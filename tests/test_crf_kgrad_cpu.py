"""The kernel-bandwidth gradient's float64 restatement (oracle/crf_kgrad_oracle.py) against central finite
differences of the frozen-lattice forward; its mutants against the same differences and against the per-case bars of
the GPU tests (tests/crf_kgrad_cases.py); its ``reference`` convention against the reference's own kernel_grad (the
live build and tests/golden/crf_kgrad_ref.npz); and the CPU-side refusals of nn.dense_crf's theta_bi / theta_sp."""
import os

import numpy as np
import pytest

import helpers
from crf_kgrad_cases import GOLDEN, GOLDEN_CASES, KgradTruth, configs, golden_inputs, label_case
from crf_compat_cases import compat_mats
from crf_grad_cases import grad_params, upstream
from oracle import crf_kgrad_oracle as K
from oracle import meanfield64

SHAPE = (9, 11)
FD_REL = 1e-4    # the analytic derivative against central differences (step 1e-5 of each sigma), relative to max|fd|;
# the worst case seen is 6e-6, the mutants and the reference's convention miss by 1e-2 and more


def _case(img, sf, M, T, seed, values=None):
    H, W = SHAPE
    image = helpers.small_image(np.random.RandomState(seed), H, W, img)
    p = helpers.make_params(values, T) if values is not None else grad_params(sf, T)
    P = meanfield64.Problem(image, p)
    unary = helpers.log_unary(1, H, W, M, seed, scale=1.0)[0]
    return K.Frozen(P, image, p), unary, upstream(H, W, M, seed + 1), p


def _fd_err(frozen, unary, G, T, mus, **kw):
    """max |analytic - fd| relative to max |fd| (absolute where the gradient vanishes: one label)."""
    th = frozen.theta0
    fd = K.finite_diff(frozen, th, unary, G, T, mus)
    got = K.theta_grad(frozen, th, unary, G, T, mus, **kw)[0]
    return float(np.abs(got - fd).max() / max(float(np.abs(fd).max()), 1.0))


CASES = ([(img, sf, M, "potts") for img in ("smooth", "noise") for sf in (1.0, 12.0) for M in (1, 2, 6, 21)
          if M in (2, 6) or sf == 1.0]
         + [(img, 1.0, 6, "nonsym") for img in ("smooth", "noise")] + [("noise", 12.0, 2, "nonsym")])


@pytest.mark.parametrize("img,sf,M,mu", CASES)
def test_theta_grad_matches_finite_differences(img, sf, M, mu):
    T = 3
    frozen, unary, G, _ = _case(img, sf, M, T, 40 + M)
    mus = None if mu == "potts" else compat_mats("nonsym", M, M + T)
    assert _fd_err(frozen, unary, G, T, mus) < FD_REL


@pytest.mark.parametrize("name", ["aniso_xy", "aniso_rgb", "weights_neg"])
def test_theta_grad_at_other_parameters(name):
    values, _, img = helpers.PARAM_SETS[name][:3]
    T = 2
    frozen, unary, G, _ = _case("smooth" if img == "smooth" else "noise", None, 6, T, 7, values)
    assert _fd_err(frozen, unary, G, T, None) < FD_REL
    assert _fd_err(frozen, unary, G, T, compat_mats("nonsym", 6, 8)) < FD_REL


def test_zero_iterations_give_zero():
    frozen, unary, G, _ = _case("noise", 1.0, 3, 0, 5)
    assert not np.any(K.theta_grad(frozen, frozen.theta0, unary, G, 0)[0])


@pytest.mark.parametrize("mutant", sorted(K.MUTANTS))
def test_mutants_miss_the_finite_differences(mutant):
    frozen, unary, G, _ = _case("noise", 1.0, 6, 3, 11)
    assert _fd_err(frozen, unary, G, 3, None, mutant=mutant) > 1e2 * FD_REL


def test_reference_convention_differentiates_the_transpose():
    """The reference's Permutohedral::gradient blurs K's order where K^T's belongs: its kernel_grad is the derivative
    of a different function, off by far more than the exact restatement's finite-difference error."""
    frozen, unary, G, _ = _case("noise", 1.0, 6, 3, 12)
    assert _fd_err(frozen, unary, G, 3, None, convention="reference") > 1e2 * FD_REL


def _golden():
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", GOLDEN))


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_reference_convention_matches_the_reference(name):
    """The oracle's ``convention="reference"`` reproduces the reference's own DenseCRF::gradient kernel_grad (the live
    build when present, and the frozen golden), while the exact derivative does not: the reference differentiates
    K^T where K is meant."""
    image, unary, G, p, mus = golden_inputs(name)
    frozen = K.Frozen(meanfield64.Problem(image, p), image, p)
    _, dp_ref, A = K.theta_grad(frozen, frozen.theta0, unary, G, int(p.n_iters), mus, convention="reference")
    _, dp_exact, _ = K.theta_grad(frozen, frozen.theta0, unary, G, int(p.n_iters), mus)
    # the reference runs in float32: a float32 sum of terms of magnitude A
    bar = K.p_in_reference_order(2.0 ** -12 * A)
    refs = [_golden()[name + "/kernel_grad"]]
    if K.ref_available():
        refs.append(K.ref_kernel_grad(image, unary, p, G, mus))
    for ref in refs:
        assert np.all(np.abs(ref - K.p_in_reference_order(dp_ref)) <= bar), (ref, K.p_in_reference_order(dp_ref))
        assert np.any(np.abs(ref - K.p_in_reference_order(dp_exact)) > 100 * bar)


@pytest.mark.parametrize("name,case", configs(), ids=[n for n, _ in configs()])
def test_mutants_outside_the_device_bars(name, case):
    """Every mutant, restated in float32, falls outside the per-case bar the GPU tests hold the device to."""
    images, p, unary, G, mus, compare = case()
    if int(p.n_iters) == 0 or unary.shape[-1] == 1:
        pytest.skip("the gradient is exactly zero: the device must return zeros (test_gpu_crf_kgrad.py)")
    b = compare[-1]
    t = KgradTruth(images[b], p, unary[b], G[b], mus)
    for mutant in sorted(K.MUTANTS):
        assert t.mutant_excess(mutant) > 1.0, mutant


def test_float32_models_within_their_bars():
    images, p, unary, G, mus, compare = label_case(6, 3)
    t = KgradTruth(images[0], p, unary[0], G[0], mus)
    for m in t.models:
        t.check(m, "model")


def test_restated_simplex_reproduces_the_build():
    """Frozen() refuses when its float32 restatement of the simplex misses one barycentric weight of the oracle's
    lattices; building it on both image kinds is the check."""
    for img in ("smooth", "noise"):
        _case(img, 12.0, 2, 1, 3)


def test_dense_crf_refuses_bad_theta():
    torch = pytest.importorskip("torch")
    from dsrg_b200 import nn
    u = torch.zeros(1, 3, 5, 6)
    im = torch.zeros(1, 5, 6, 3, dtype=torch.uint8)
    bad = [dict(theta_bi=torch.ones(4)), dict(theta_sp=torch.ones(3)), dict(theta_bi=torch.ones(5, dtype=torch.int64)),
           dict(theta_sp=[1.0, 2.0]), dict(theta_sp=torch.tensor([1.0, 0.0])), dict(theta_sp=torch.tensor([1.0, -2.0])),
           dict(theta_bi=torch.tensor([1.0, 2.0, float("nan"), 1.0, 1.0])),
           dict(theta_bi=torch.tensor([1.0, 2.0, float("inf"), 1.0, 1.0]))]
    for kw in bad:
        with pytest.raises(ValueError, match="theta"):
            nn.dense_crf(u, im, **kw)
