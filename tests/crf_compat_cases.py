"""Cases and the per-case bar of the compatibility-matrix CRF tests (test_crf_compat_cpu.py, test_gpu_crf_compat.py).

The truth is oracle/crf_compat_oracle in float64.  A case's bar is built like crf_grad_cases.GradTruth's: BAR_K times
the largest error of the float32 models (the oracle's sequential splat, shuffled splat orders, the device's own
operation order including the mat-vec), each run forward and backward in float32.  Floors:
* marginals and dL/dunary: BAR_FLOOR times their scale (1, and max(|G|, |dL/dU|)), for cases whose models agree
  exactly (M = 1, or mu = 0 and T = 0).
* dL/dmu: 2^-14 times the entry's sum of |S_k|·|Q_t|.  The device sums an entry's terms in float32 sequentially over a
  tile's 256 pixels, then over the iterations, then over the tiles (451 at 321 x 321, at most 12 in these cases), so
  its rounding error is below (256 + 10 + 451)·2^-24 < 2^-14 of that sum.
"""
import numpy as np

import helpers
from oracle import crf_compat_oracle

COMPAT_ITERS = (0, 1, 2, 3, 10)
COMPAT_M = [1, 2, 6, 21, 24, 32]
COMPAT_FLOOR = 2.0 ** -14
GOLDEN = "crf_compat_grad_ref.npz"


def compat_mats(kind, M, seed, w1=10.0, w2=3.0):
    """(mu_bi, mu_sp) float32 (M, M): "zero", "potts" (-w I), "sym" (random symmetric), "diag" (distinct diagonal),
    "classic" (w (1 - I)), "nonsym" (random, not symmetric)."""
    rng = np.random.RandomState(seed)
    eye = np.eye(M)
    if kind == "zero":
        m = [np.zeros((M, M)), np.zeros((M, M))]
    elif kind == "potts":
        m = [-w1 * eye, -w2 * eye]
    elif kind == "classic":
        m = [w1 * (1 - eye), w2 * (1 - eye)]
    elif kind == "diag":
        m = [np.diag(-w1 * (0.5 + rng.rand(M))), np.diag(-w2 * (0.5 + rng.rand(M)))]
    else:
        m = [s * (rng.randn(M, M) - 2 * eye) for s in (3.0, 1.0)]
        if kind == "sym":
            m = [0.5 * (x + x.T) for x in m]
        else:
            assert kind == "nonsym"
    return tuple(np.asarray(x, np.float32) for x in m)


class CompatTruth(object):
    """float64 marginals and gradients of one image's case and their bars; .models holds every float32 model's
    (Q_T, dL/dU, dL/dmu)."""

    def __init__(self, problem, unary, G, T, mus, models=helpers.BAR_MODELS, mutants=()):
        self.T = T
        q64 = crf_compat_oracle.run(problem, unary, mus, T)
        self.q = q64[T]
        self.gU, self.gmu, self.amu = crf_compat_oracle.backward(problem, q64, G, mus)
        self.models = []
        for m in models:
            kw = dict(m)
            exp_seed = kw.pop("exp_seed", 0)
            q32 = crf_compat_oracle.run(problem, unary, mus, T, np.float32, exp_seed=exp_seed, **kw)
            gu, gm, _ = crf_compat_oracle.backward(problem, q32, G, mus, np.float32, **kw)
            self.models.append((q32[T], gu, gm))
        err_q = max([float(np.abs(q - self.q).max()) for q, _, _ in self.models] + [0.0])
        err_u = max([float(np.abs(u - self.gU).max()) for _, u, _ in self.models] + [0.0])
        err_mu = np.max([np.abs(g - self.gmu) for _, _, g in self.models] + [np.zeros_like(self.gmu)], axis=0)
        self.scale = max(float(np.abs(G).max()), float(np.abs(self.gU).max()))
        self.bar_q = max(helpers.BAR_K * err_q, helpers.BAR_FLOOR)
        self.bar_u = max(helpers.BAR_K * err_u, helpers.BAR_FLOOR * self.scale)
        self.bar_mu = np.maximum(helpers.BAR_K * err_mu, COMPAT_FLOOR * self.amu)
        self.err_u = err_u
        self.mutants = {}
        if mutants:
            q32 = crf_compat_oracle.run(problem, unary, mus, T, np.float32)
            for name in mutants:
                self.mutants[name] = crf_compat_oracle.backward(problem, q32, G, mus, np.float32, mutant=name)[:2]

    def over(self, gU, gmu):
        """The largest error over its bar, of dL/dU and of dL/dmu."""
        return (float(np.abs(gU - self.gU).max()) / self.bar_u,
                float((np.abs(np.asarray(gmu, np.float64) - self.gmu) / self.bar_mu).max()))

    def check(self, q, gU, gmu, what=""):
        if q is not None:
            e = float(np.abs(q - self.q).max())
            assert e <= self.bar_q, "%s marginals off by %.3g > bar %.3g" % (what, e, self.bar_q)
        e = float(np.abs(gU - self.gU).max())
        assert e <= self.bar_u, "%s dL/dunary off by %.3g > bar %.3g (float32 models %.3g, scale %.3g)" % (
            what, e, self.bar_u, self.err_u, self.scale)
        if gmu is not None:
            d = np.abs(np.asarray(gmu, np.float64) - self.gmu) - self.bar_mu
            i = np.unravel_index(int(np.argmax(d)), d.shape)
            assert d[i] <= 0, "%s dL/dmu%s = %.9g, float64 %.9g: off by %.3g > bar %.3g" % (
                what, i, gmu[i], self.gmu[i], abs(gmu[i] - self.gmu[i]), self.bar_mu[i])


# the cases of the frozen reference results (tests/golden/make_crf_compat_golden.py), all with symmetric mu (the
# reference symmetrises): name -> (H, W, image, M, scale factor, T, seed, mu kind)
GOLDEN_CASES = {
    "tiny_sym": (7, 9, "noise", 4, 1.0, 5, 3, "sym"),
    "smooth_diag": (37, 45, "smooth", 21, 1.0, 3, 5, "diag"),
    "noise_classic": (41, 41, "noise", 6, 12.0, 10, 7, "classic"),
}


def golden_inputs(name):
    """(image (H, W, 3), unary (H, W, M), G (H, W, M), params, (mu_bi, mu_sp)) of a golden case."""
    from crf_grad_cases import grad_params, upstream
    H, W, img, M, sf, T, seed, kind = GOLDEN_CASES[name]
    image = helpers.small_image(np.random.RandomState(seed), H, W, img)
    unary = helpers.log_unary(1, H, W, M, seed, scale=1.0)[0]
    return image, unary, upstream(H, W, M, seed), grad_params(sf, T), compat_mats(kind, M, seed)
