"""The CRF gradient's float64 restatement (oracle/crf_grad_oracle.backward) against the reference's own
DenseCRF::gradient (densecrf.cpp:238-297) and against central finite differences of the float64 forward; its float32
models against their bar; and the bar against a backward that blurs K^T in K's axis order.  No GPU."""
import os

import numpy as np
import pytest

import helpers
from crf_grad_cases import GOLDEN, GOLDEN_CASES, GRAD_ITERS, GRAD_M, GradTruth, golden_inputs, grad_params, upstream
from oracle import crf_grad_oracle, meanfield64

GOLDEN_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", GOLDEN)


def _case(H, W, img, M, sf, T, seed, zero=None):
    image = helpers.small_image(np.random.RandomState(seed), H, W, img)
    unary = helpers.log_unary(1, H, W, M, seed, scale=1.0)[0]
    p = grad_params(sf, T, zero)
    return meanfield64.Problem(image, p), image, unary, upstream(H, W, M, seed), p


@pytest.mark.parametrize("name", sorted(GOLDEN_CASES))
def test_float64_backward_matches_the_reference_gradient(name):
    """The reference computes its gradient in float32 (its forward and backward), so it lies within the float32
    models' bar of the float64 truth; where oracle/_ref is built its live result must also equal the frozen one."""
    image, unary, G, p = golden_inputs(name)
    truth = GradTruth(meanfield64.Problem(image, p), unary, G, p.n_iters)
    with np.load(GOLDEN_PATH) as z:
        gU, gw = z[name + "/grad_unary"], z[name + "/grad_potts"]
    if crf_grad_oracle.ref_available():
        live_u, live_w = crf_grad_oracle.ref_crf_gradient(image, unary, p, G)
        np.testing.assert_array_equal(live_u, gU)
        np.testing.assert_array_equal(np.array(live_w), gw)
    truth.check(gU, gw, "reference %s:" % name)
    # the gradients are not vanishing: the comparison above is not of two zeros
    assert np.abs(truth.gU).max() > 1e-3 and min(abs(w) for w in truth.gw) > 1e-6


@pytest.mark.parametrize("T", [1, 3])
def test_float64_backward_matches_finite_differences(T):
    """L = <G, Q_T>: central differences of the float64 forward in a few unaries and in both Potts weights."""
    P, image, unary, G, p = _case(7, 9, "noise", 4, 1.0, T, 3)
    gU, gw, _ = crf_grad_oracle.backward(P, P.run(unary, T), G)

    def loss(u):
        return float((P.run(u, T)[-1] * G).sum())

    rng = np.random.RandomState(1)
    for _ in range(4):
        i = tuple(rng.randint(s) for s in unary.shape)
        up, um = unary.copy(), unary.copy()
        up[i] += np.float32(1e-2)
        um[i] -= np.float32(1e-2)
        fd = (loss(up) - loss(um)) / (float(up[i]) - float(um[i]))
        assert abs(fd - gU[i]) <= 1e-4 * np.abs(gU).max() + 1e-9, (i, fd, gU[i])
    for k, wi in ((1, 0), (0, 1)):   # lattice 1 is w1's (bilateral), lattice 0 w2's (spatial)
        L = P.lattices[k]
        w0, h = L.w, 1e-4
        L.w = w0 + h
        a = loss(unary)
        L.w = w0 - h
        b = loss(unary)
        L.w = w0
        fd = (a - b) / (2 * h)
        assert abs(fd - gw[wi]) <= 1e-5 * abs(gw[wi]) + 1e-9, (wi, fd, gw[wi])


CPU_CASES = ([("smooth", M, 1.0, 3, None) for M in GRAD_M] + [("noise", 21, 1.0, T, None) for T in GRAD_ITERS]
             + [("smooth", 6, 12.0, 2, z) for z in ("w1", "w2")])


@pytest.mark.parametrize("img,M,sf,T,zero", CPU_CASES)
def test_float32_models_lie_within_the_bar_and_the_mutant_beyond(img, M, sf, T, zero):
    H, W = helpers.FUSED_SHAPES[img]
    H, W = H // 2, W // 2
    P, _, unary, G, p = _case(H, W, img, M, sf, T, 11 + M, zero)
    truth = GradTruth(P, unary, G, T, mutant="transpose_forward_order")
    for k, (u, w) in enumerate(truth.models):
        truth.check(u, w, "model %d:" % k)
    # the bar is float32 noise, well below the gradient itself (M = 1 has none: Q is 1 and g is 0).  Ten iterations on
    # a noise image amplify it most: there the bar came to 0.9 % of the gradient's scale (206)
    if M > 1:
        assert truth.bar_u <= 2e-2 * truth.scale, (truth.bar_u, truth.scale)
    if zero is not None:
        assert truth.gw[0 if zero == "w1" else 1] != 0.0   # a zeroed weight still has a gradient
    if T == 0:
        assert truth.gw == (0.0, 0.0)
    if T == 0 or M == 1:
        return
    # K^T blurred in K's order (0..d) is a different operator: the bar sees it, on dL/dunary or a Potts weight
    mu, mw = truth.mutant
    over = [float(np.abs(mu - truth.gU).max()) / truth.bar_u] + \
        [abs(mw[i] - truth.gw[i]) / truth.bar_w[i] for i in (0, 1)]
    assert max(over) > 1.0, "the transposed blur in forward order stays within the bar: %s" % over


@pytest.mark.parametrize("H,W,img", helpers.MF64_TINY)
def test_phantom_lane_shapes(H, W, img):
    """N % 4 = 0..3: the phantom lanes' vertices are real rows of the backward's lattices too."""
    P, _, unary, G, p = _case(H, W, img, helpers.MF64_TINY_M, 1.0, 3, helpers.MF64_TINY_SEED)
    truth = GradTruth(P, unary, G, 3)
    for u, w in truth.models:
        truth.check(u, w)
    if crf_grad_oracle.ref_available():
        image = helpers.small_image(np.random.RandomState(helpers.MF64_TINY_SEED), H, W, img)
        ru, rw = crf_grad_oracle.ref_crf_gradient(image, unary, p, G)
        truth.check(ru, rw, "reference:")


def test_zero_iterations_is_the_softmax_jacobian():
    P, _, unary, G, p = _case(5, 6, "noise", 6, 1.0, 0, 2)
    gU, gw, _ = crf_grad_oracle.backward(P, P.run(unary, 0), G)
    q = P.run(unary, 0)[0]
    np.testing.assert_allclose(gU, q * (G - (G * q).sum(-1, keepdims=True)), rtol=1e-12, atol=1e-15)
    assert gw == (0.0, 0.0)
