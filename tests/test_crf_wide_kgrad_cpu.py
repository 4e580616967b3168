"""The kernel-bandwidth and feature gradients' float64 restatements (oracle/crf_kgrad_oracle.py,
oracle/crf_fgrad_oracle.py) above 32 labels: against central finite differences at 33 and 81 labels with Potts terms
and matrices; their ``reference`` convention against the reference's own kernel_grad at those counts (the live build
and tests/golden/crf_wide_kgrad_ref.npz); every oracle mutant outside the bars of tests/crf_wide_kgrad_cases.py in the
cases the GPU file runs; and nn.dense_crf_wide's refusals of the new arguments that need no GPU."""
import os

import numpy as np
import pytest

import helpers
from crf_compat_cases import compat_mats
from crf_fgrad_cases import features_of
from crf_grad_cases import grad_params, upstream
from crf_wide_kgrad_cases import (GOLDEN, GOLDEN_CASES, WideFgradTruth, WideKgradTruth, configs, golden_inputs,
                                  wide_floor)
from oracle import crf_fgrad_oracle as F
from oracle import crf_kgrad_oracle as K
from oracle import meanfield64

FD_REL = 1e-4   # as test_crf_kgrad_cpu.py: the analytic derivative against central differences, relative to max|fd|


def _inputs(M, T, seed, img="noise", H=9, W=11):
    image = helpers.small_image(np.random.RandomState(seed), H, W, img)
    unary = helpers.log_unary(1, H, W, M, seed, scale=1.0)[0]
    return image, grad_params(1.0, T), unary, upstream(H, W, M, seed + 1)


@pytest.mark.parametrize("M", [33, 81])
@pytest.mark.parametrize("mu", [None, "nonsym"])
def test_theta_restatement_meets_finite_differences(M, mu):
    T = 2
    image, p, unary, G = _inputs(M, T, 40 + M)
    frozen = K.Frozen(meanfield64.Problem(image, p), image, p)
    mus = compat_mats(mu, M, M) if mu else None
    fd = K.finite_diff(frozen, frozen.theta0, unary, G, T, mus)
    got = K.theta_grad(frozen, frozen.theta0, unary, G, T, mus)[0]
    assert np.abs(got - fd).max() < FD_REL * max(float(np.abs(fd).max()), 1.0), (got, fd)


@pytest.mark.parametrize("M", [33, 81])
@pytest.mark.parametrize("mu", [None, "nonsym"])
def test_feature_restatement_meets_finite_differences(M, mu):
    image, p, unary, G = _inputs(M, 2, 50 + M, img="photo")
    f = features_of("guide", image, p, M)
    mus = compat_mats(mu, M, M + 1) if mu else None
    fz = F.Frozen(F.FeatProblem(f, p))
    df = F.feature_grad(fz, unary, G, mus)[0]
    d = np.random.RandomState(M).randn(*df.shape)   # every pixel and channel at once
    fd = F.finite_diff(fz, unary, G, d, mus)
    assert abs(fd - (df * d).sum()) <= 1e-6 * max(1.0, abs(fd)), (fd, (df * d).sum())


def _golden():
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", GOLDEN))


@pytest.mark.parametrize("name", sorted(GOLDEN_CASES))
def test_reference_convention_matches_the_reference(name):
    """The oracles' ``convention="reference"`` reproduce the reference's own kernel_grad above 32 labels (the live
    build when present, and the frozen golden); the exact derivatives do not (the reference differentiates K^T where K
    is meant: off by more than ten bars).  The reference sums in float32, over deeper label chains than at 21 labels:
    the bar is the float32 one of test_crf_kgrad_cpu.py scaled by wide_floor(M) / wide_floor(32)."""
    image, feats, unary, G, p, mus, kind = golden_inputs(name)
    M = unary.shape[-1]
    scale = wide_floor(M) / wide_floor(32)
    refs = [_golden()[name + "/kernel_grad"]]
    if kind == "theta":
        frozen = K.Frozen(meanfield64.Problem(image, p), image, p)
        _, dp_ref, A = K.theta_grad(frozen, frozen.theta0, unary, G, int(p.n_iters), mus, convention="reference")
        _, dp_exact, _ = K.theta_grad(frozen, frozen.theta0, unary, G, int(p.n_iters), mus)
        bar = K.p_in_reference_order(2.0 ** -12 * scale * A)
        if K.ref_available():
            refs.append(K.ref_kernel_grad(image, unary, p, G, mus))
        for ref in refs:
            assert np.all(np.abs(ref - K.p_in_reference_order(dp_ref)) <= bar), (ref, K.p_in_reference_order(dp_ref))
            assert np.any(np.abs(ref - K.p_in_reference_order(dp_exact)) > 10 * bar)
    else:
        fz = F.Frozen(F.FeatProblem(feats, p))
        d_ref, dsp_ref, mag = F.feature_grad(fz, unary, G, mus, convention="reference")
        d_exact = F.feature_grad(fz, unary, G, mus)[0]
        want = F.full_kernel_grad(d_ref, feats)
        bar = 2.0 ** -12 * scale * F.full_kernel_grad(mag, np.abs(feats))
        dp_sp = -dsp_ref * fz.theta_sp
        if F.ref_available():
            refs.append(F.ref_full_kernel_grad(feats, unary, p, G, mus))
        for ref in refs:
            assert np.all(np.abs(ref[2:] - want) <= bar), (ref[2:], want)
            assert np.allclose(ref[:2], dp_sp, rtol=1e-4, atol=1e-6 * np.abs(dp_sp).max())
            assert np.any(np.abs(ref[2:] - F.full_kernel_grad(d_exact, feats)) > 10 * bar)


@pytest.mark.parametrize("name,case,kind", configs(), ids=[c[0] for c in configs()])
def test_mutants_outside_the_device_bars(name, case, kind):
    """Every oracle mutant, restated in float32, falls outside the bar the GPU file holds the device to."""
    c = case()
    p = c[2] if kind == "feat" else c[1]
    if int(p.n_iters) == 0:
        pytest.skip("the gradient is exactly zero: the device must return zeros (test_gpu_crf_wide_kgrad.py)")
    if kind == "feat":
        images, feats, p, unary, G, mus = c
        t = WideFgradTruth(feats[1], p, unary[1], G[1], mus)
    else:
        images, p, unary, G, mus = c
        t = WideKgradTruth(images[1], p, unary[1], G[1], mus)
    for mutant in sorted(K.MUTANTS):
        assert t.mutant_excess(mutant) > 1.0, mutant


def test_bars_hold_the_float32_models():
    image, p, unary, G = _inputs(81, 3, 5)
    t = WideKgradTruth(image, p, unary, G)
    for m in t.models:
        t.check(m, "model")


def test_dense_crf_wide_refuses_bad_theta_and_features():
    torch = pytest.importorskip("torch")
    from dsrg_b200 import nn
    u = torch.zeros(2, 40, 4, 5)
    f = torch.zeros(2, 5, 4, 5)
    image = torch.zeros(2, 4, 5, 3, dtype=torch.uint8)
    with pytest.raises(ValueError, match="image is not used"):
        nn.dense_crf_wide(u, image, features_bi=f)
    with pytest.raises(ValueError, match="theta_bi and features_bi"):
        nn.dense_crf_wide(u, None, features_bi=f, theta_bi=torch.ones(5))
    for bad in (torch.zeros(2, 4, 4, 5), torch.zeros(2, 5, 4, 5, dtype=torch.float64), torch.zeros(1, 5, 4, 5),
                np.zeros((2, 5, 4, 5), np.float32)):
        with pytest.raises(ValueError, match="features_bi must be"):
            nn.dense_crf_wide(u, None, features_bi=bad)
    for kw in (dict(theta_bi=torch.ones(4)), dict(theta_sp=torch.ones(3)), dict(theta_sp=torch.tensor([1.0, 0.0])),
               dict(theta_bi=torch.tensor([1.0, 2.0, float("nan"), 1.0, 1.0])), dict(theta_sp=[1.0, 2.0])):
        with pytest.raises(ValueError, match="theta"):
            nn.dense_crf_wide(u, image, **kw)
    with pytest.raises(ValueError, match="CUDA"):   # well-formed, but the CRF runs on the device only
        nn.dense_crf_wide(u, None, features_bi=f)
    with pytest.raises(ValueError, match="CUDA"):
        nn.dense_crf_wide(u, image, theta_sp=torch.ones(2))
