"""Cases and the per-case bar of the CRF gradient tests (test_crf_grad_cpu.py, test_gpu_crf_grad.py).

The truth is oracle/crf_grad_oracle.backward in float64 on the float64 forward's iterates.  A case's bar is built
like helpers.mf64_truth_and_bar's: BAR_K times the largest error of the float32 models (the oracle's sequential splat,
shuffled splat orders, the device's own operation order), each run forward and backward in float32, so the bar is
the float32 noise of this very case.  Floors:
* dL/dunary: BAR_FLOOR times the scale max(|G|, |dL/dU|), for cases whose models agree exactly (M = 1 gives 0).
* Potts: 2^-16 times the sum of |S_k|·|Q_t| over the gradient's terms.  The device sums them in float32 in a tree
  of depth below 64 (a thread's labels, a warp, the tile's warps, the iterations, the tiles), so its rounding error is
  below 64·2^-24 = 2^-18 of that sum; the floor is four times that.
"""
import numpy as np

import helpers
from oracle import crf_grad_oracle

GRAD_ITERS = (0, 1, 2, 3, 10)
GRAD_M = [1, 2, 6, 21, 24, 32]
POTTS_FLOOR = 2.0 ** -16
GOLDEN = "crf_grad_ref.npz"


def upstream(H, W, M, seed):
    """(H, W, M) float32 dL/dQ_T: a smooth field plus noise, like a loss's gradient."""
    rng = np.random.RandomState(seed)
    return (rng.randn(H, W, M) + np.linspace(-1, 1, M)[None, None, :]).astype(np.float32)


def grad_params(sf, T, zero=None, w1=None, w2=None):
    p = helpers.mf64_problem_params(sf, zero, T)
    if w1 is not None:
        p.w1 = w1
    if w2 is not None:
        p.w2 = w2
    return p


class GradTruth(object):
    """float64 gradients of one image's case and their bars; .models holds every float32 model's result."""

    def __init__(self, problem, unary, G, T, models=helpers.BAR_MODELS, mutant=None):
        self.T = T
        q64 = problem.run(unary, T)
        self.gU, self.gw, self.gabs = crf_grad_oracle.backward(problem, q64, G)
        self.q64 = q64
        self.models = []
        for m in models:
            kw = dict(m)
            exp_seed = kw.pop("exp_seed", 0)
            q32 = problem.run(unary, T, np.float32, exp_seed=exp_seed, **kw)
            self.models.append(crf_grad_oracle.backward(problem, q32, G, np.float32, **kw)[:2])
        err_u = max([float(np.abs(u - self.gU).max()) for u, _ in self.models] + [0.0])
        err_w = [max([abs(w[i] - self.gw[i]) for _, w in self.models] + [0.0]) for i in (0, 1)]
        scale = max(float(np.abs(G).max()), float(np.abs(self.gU).max()))
        self.bar_u = max(helpers.BAR_K * err_u, helpers.BAR_FLOOR * scale)
        self.bar_w = [max(helpers.BAR_K * err_w[i], POTTS_FLOOR * self.gabs[i]) for i in (0, 1)]
        self.err_u, self.err_w, self.scale = err_u, err_w, scale
        if mutant:
            q32 = problem.run(unary, T, np.float32)
            self.mutant = crf_grad_oracle.backward(problem, q32, G, np.float32, mutant=mutant)[:2]

    def check(self, gU, gw, what=""):
        e = float(np.abs(gU - self.gU).max())
        assert e <= self.bar_u, "%s dL/dunary off by %.3g > bar %.3g (float32 models %.3g, scale %.3g)" % (
            what, e, self.bar_u, self.err_u, self.scale)
        if gw is not None:
            for i, name in ((0, "w1"), (1, "w2")):
                ew = abs(float(gw[i]) - self.gw[i])
                assert ew <= self.bar_w[i], "%s dL/d%s = %.9g, float64 %.9g: off by %.3g > bar %.3g" % (
                    what, name, gw[i], self.gw[i], ew, self.bar_w[i])


# the cases of the frozen reference gradients (tests/golden/make_crf_grad_golden.py):
# name -> (H, W, image, M, scale factor, T, seed)
GOLDEN_CASES = {
    "tiny_noise": (7, 9, "noise", 4, 1.0, 5, 3),
    "smooth_21": (37, 45, "smooth", 21, 1.0, 3, 5),
    "noise_sf12": (41, 41, "noise", 6, 12.0, 10, 7),
}


def golden_inputs(name):
    """(image (H, W, 3), unary (H, W, M), G (H, W, M), params) of a golden case."""
    H, W, img, M, sf, T, seed = GOLDEN_CASES[name]
    image = helpers.small_image(np.random.RandomState(seed), H, W, img)
    unary = helpers.log_unary(1, H, W, M, seed, scale=1.0)[0]
    return image, unary, upstream(H, W, M, seed), grad_params(sf, T)
