"""The per-pixel feature gradient's float64 restatement (oracle/crf_fgrad_oracle.py) without a GPU: against central
finite differences of the frozen-simplex forward, against the kernel-bandwidth oracle through the identity
sum_i f_i dL/df_i = dL/dp, every mutant outside the device's bars, and nn.dense_crf's refusals of features_bi."""
import os

import numpy as np
import pytest

import helpers
from crf_compat_cases import compat_mats
from crf_fgrad_cases import GOLDEN, GOLDEN_CASES, FEATURE_KINDS, FgradTruth, case, features_of, golden_inputs, inputs
from crf_grad_cases import grad_params
from oracle import crf_fgrad_oracle as F
from oracle import crf_kgrad_oracle as K
from oracle import meanfield64


def _tiny(kind, mu=None, T=2, M=3, seed=0):
    H, W = 5, 6
    image = helpers.small_image(np.random.RandomState(40 + seed), H, W, "noise")
    p = grad_params(1.0, T)
    f = features_of(kind, image, p, seed)
    unary, G = inputs(1, H, W, M, 60 + seed)
    return image, f, p, unary[0], G[0], (compat_mats(mu, M, 5) if mu else None)


@pytest.mark.parametrize("kind", FEATURE_KINDS)
@pytest.mark.parametrize("mu", [None, "nonsym"])
def test_restatement_matches_finite_differences(kind, mu):
    _, f, p, unary, G, mus = _tiny(kind, mu)
    fz = F.Frozen(F.FeatProblem(f, p))
    df, _, _ = F.feature_grad(fz, unary, G, mus)
    rng = np.random.RandomState(7)
    for _ in range(2):   # random directions: every pixel and channel at once
        d = rng.randn(*df.shape)
        fd = F.finite_diff(fz, unary, G, d, mus)
        assert abs(fd - (df * d).sum()) <= 1e-6 * max(1.0, abs(fd)), (fd, (df * d).sum())
    for pix, c in ((0, 0), (7, 3), (29, 4)):   # single entries, the last pixel included
        d = np.zeros_like(df)
        d[pix, c] = 1.0
        fd = F.finite_diff(fz, unary, G, d, mus)
        assert abs(fd - df[pix, c]) <= 1e-6 * max(1.0, abs(fd)), (pix, c, fd, df[pix, c])


@pytest.mark.parametrize("mu", [None, "nonsym"])
def test_features_of_the_image_give_the_theta_gradient(mu):
    """With f = float32(x)/theta_alpha, ... the lattice is the image path's, and sum f . dL/df is its dL/dp."""
    image, f, p, unary, G, mus = _tiny("image", mu, T=3)
    fz = F.Frozen(F.FeatProblem(f, p))
    img_problem = meanfield64.Problem(image, p)
    for a, b in zip(fz.problem.lattices, img_problem.lattices):
        assert np.array_equal(a.bary, b.bary) and np.array_equal(a.offset, b.offset)
    df, dsp, _ = F.feature_grad(fz, unary, G, mus)
    kfz = K.Frozen(img_problem, image, p)
    dth, dp, _ = K.theta_grad(kfz, kfz.theta0, unary, G, 3, mus)
    # the kernel-bandwidth truth sits at the float64 x/theta, this one at its float32 rounding: 1e-5 apart here
    got = (f.reshape(-1, 5).astype(np.float64) * df).sum(0)
    assert np.allclose(got, dp[0:5], rtol=1e-4, atol=1e-9 * np.abs(dp).max()), (got, dp[0:5])
    assert np.allclose(dsp, dth[5:7], rtol=1e-4, atol=0), (dsp, dth[5:7])


def test_reference_convention_differs_from_exact():
    """The reference's K^T convention is a different number wherever a blur neighbour is missing."""
    _, f, p, unary, G, mus = _tiny("random")
    fz = F.Frozen(F.FeatProblem(f, p))
    exact = F.feature_grad(fz, unary, G)[0]
    ref = F.feature_grad(fz, unary, G, convention="reference")[0]
    assert np.abs(exact - ref).max() > 1e-3 * np.abs(exact).max()


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_reference_convention_matches_the_reference_full_kernel(name):
    """The oracle's ``convention="reference"`` dL/df, taken to dL/dP = fg f^T, reproduces the reference's own
    kernel_grad of a FULL_KERNEL term at P = I (the live build when present, and the frozen golden); the exact
    derivative does not (the reference differentiates K^T where K is meant)."""
    features, unary, G, p, mus = golden_inputs(name)
    fz = F.Frozen(F.FeatProblem(features, p))
    d_ref, dsp_ref, mag = F.feature_grad(fz, unary, G, mus, convention="reference")
    d_exact = F.feature_grad(fz, unary, G, mus)[0]
    want = F.full_kernel_grad(d_ref, features)
    # the reference runs in float32: a float32 sum of terms of magnitude |f| times mag
    bar = 2.0 ** -12 * F.full_kernel_grad(mag, np.abs(features))
    dp_sp = -dsp_ref * fz.theta_sp
    refs = [np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", GOLDEN))[name + "/kernel_grad"]]
    if F.ref_available():
        refs.append(F.ref_full_kernel_grad(features, unary, p, G, mus))
    for ref in refs:
        assert np.all(np.abs(ref[2:] - want) <= bar), (ref[2:], want)
        assert np.allclose(ref[:2], dp_sp, rtol=1e-4, atol=1e-6 * np.abs(dp_sp).max())
        assert np.any(np.abs(ref[2:] - F.full_kernel_grad(d_exact, features)) > 100 * bar)


@pytest.mark.parametrize("mutant", sorted(F.MUTANTS))
@pytest.mark.parametrize("kind", FEATURE_KINDS)
def test_mutants_fall_outside_the_bars(mutant, kind):
    images, feats, p, unary, G, mus = case("noise", 1.0, kind, 6, 3, H=9, W=11, seed=3)
    t = FgradTruth(feats[0], p, unary[0], G[0], mus)
    assert t.mutant_excess(mutant) > 1.0


def test_bars_hold_the_float32_models():
    images, feats, p, unary, G, mus = case("noise", 1.0, "guide", 6, 3, H=9, W=11, seed=4)
    t = FgradTruth(feats[0], p, unary[0], G[0], mus)
    df = F.feature_grad(t.fz, unary[0], G[0], dtype=np.float32, splat_order=9)[0]
    t.check(df)


def test_random_features_fill_the_hash_capacity():
    """The engine's hash holds (d+1)(N+P) vertex ids in 2(d+1)(N+P) slots per image (api.cu: lattice_shape): random
    features can give every incidence its own vertex and still fit."""
    H, W = 13, 17
    f = np.random.RandomState(1).uniform(-140, 140, (H * W, 5)).astype(np.float32)
    lat = F.crf_oracle.OracleLattice(f)
    N, P = H * W, (4 - (H * W) % 4) % 4
    assert lat.M > 0.9 * 6 * N            # nearly every incidence is a vertex of its own
    assert lat.M <= 6 * (N + P)           # capv
    assert np.abs(F.simplex(f)[1]).max() + 6 < 2047   # and the keys of +-140 fit the 12-bit range


def _torch():
    return pytest.importorskip("torch")


def test_dense_crf_refusals_without_gpu():
    torch = _torch()
    from dsrg_b200 import nn
    u = torch.zeros(2, 3, 4, 5)
    f = torch.zeros(2, 5, 4, 5)
    image = torch.zeros(2, 4, 5, 3, dtype=torch.uint8)
    with pytest.raises(ValueError, match="image is not used"):
        nn.dense_crf(u, image, features_bi=f)
    with pytest.raises(ValueError, match="theta_bi and features_bi"):
        nn.dense_crf(u, None, features_bi=f, theta_bi=torch.ones(5))
    for bad in (torch.zeros(2, 4, 4, 5), torch.zeros(2, 5, 4, 5, dtype=torch.float64), torch.zeros(1, 5, 4, 5),
                np.zeros((2, 5, 4, 5), np.float32)):
        with pytest.raises(ValueError, match="features_bi must be"):
            nn.dense_crf(u, None, features_bi=bad)
    with pytest.raises(ValueError, match="CUDA"):   # well-formed, but the CRF runs on the device only
        nn.dense_crf(u, None, features_bi=f)
    with pytest.raises(ValueError, match="image must be"):   # without features the image stays required
        nn.dense_crf(u, None)
