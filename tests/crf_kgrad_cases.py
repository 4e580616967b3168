"""Cases and the per-case bar of the kernel-bandwidth gradient tests (test_crf_kgrad_cpu.py, test_gpu_crf_kgrad.py).

The truth is oracle/crf_kgrad_oracle.theta_grad in float64 on the frozen lattices.  A case's bar is built like
crf_grad_cases.GradTruth's: BAR_K times the largest error of the float32 models (helpers.BAR_MODELS: the oracle's
sequential splat, shuffled splat orders, the device's own forward arithmetic), each run forward and backward in float32,
so the bar is the float32 noise of this very case.  Floor: KGRAD_FLOOR times A_i / theta_i, with A_i the sum over the
pixels of |f_i| times the magnitude of the terms of (dL/df)_i before they cancel.  The device sums those terms in
float32 in a tree of depth below 64 (a pixel's incidences and labels, a warp, the block's warps, the iterations, the
blocks), so its rounding error is below 64·2^-24 = 2^-18 of that sum; the floor is four times that.

CONFIGS are the cases the GPU tests run, so that the CPU tests can show every mutant outside the bars the device is
held to (the cases with one label or no iteration have a gradient of exactly zero, which no mutant changes).
"""
import numpy as np

import helpers
from crf_compat_cases import compat_mats
from crf_grad_cases import grad_params, upstream
from oracle import crf_kgrad_oracle as K
from oracle import meanfield64

KGRAD_FLOOR = 2.0 ** -16
GOLDEN = "crf_kgrad_ref.npz"


class KgradTruth(object):
    """float64 dL/dtheta of one image's case and its bar; .models holds every float32 model's result."""

    def __init__(self, image, params, unary, G, mus=None, models=helpers.BAR_MODELS):
        self.frozen = K.Frozen(meanfield64.Problem(image, params), image, params)
        self.th = self.frozen.theta0
        self.T, self.mus, self.unary, self.G = int(params.n_iters), mus, unary, G
        self.want, _, self.A = K.theta_grad(self.frozen, self.th, unary, G, self.T, mus)
        self.models = []
        for m in models:
            kw = dict(m)
            es = kw.pop("exp_seed", 0)
            self.models.append(K.theta_grad(self.frozen, self.th, unary, G, self.T, mus, dtype=np.float32,
                                            exp_seed=es, **kw)[0])
        self.err = np.max([np.abs(m - self.want) for m in self.models] + [np.zeros(7)], axis=0)
        self.bar = np.maximum(helpers.BAR_K * self.err, KGRAD_FLOOR * self.A / self.th)

    def check(self, got, what=""):
        err = np.abs(np.asarray(got, np.float64) - self.want)
        assert np.all(np.isfinite(got)), "%s %s" % (what, got)
        assert np.all(err <= self.bar), "%s err %s bar %s got %s want %s" % (what, err, self.bar, got, self.want)

    def mutant_excess(self, mutant):
        """max_i |mutant_i - want_i| / bar_i for the float32 restatement with `mutant` (> 1: outside the bar)."""
        got = K.theta_grad(self.frozen, self.th, self.unary, self.G, self.T, self.mus, mutant=mutant,
                           dtype=np.float32)[0]
        return float(np.max(np.abs(got - self.want) / np.maximum(self.bar, 1e-300)))


def inputs(images, M, seed):
    B, H, W = images.shape[:3]
    return helpers.log_unary(B, H, W, M, seed, scale=1.0), np.stack([upstream(H, W, M, seed + b) for b in range(B)])


def tiny_images(M):
    H, W = helpers.PARAM_TINY if M <= 6 else (13, 17)
    return np.stack([helpers.small_image(np.random.RandomState(70 + b), H, W, "noise") for b in range(2)])


SET_NAMES = ("aniso_xy", "aniso_rgb", "weights_neg", "decoupled_sp_direct_bi_smem")
SET_MU = ("potts_host", "potts_dev", "nonsym")
PATH_MT = ((6, 3), (21, 2), (32, 1))
LABELS = (1, 2, 6, 21, 24, 32)
ITERS = (0, 1, 2, 3, 10)


def label_case_runs(M, T):
    return T < 10 or M in (2, 21)


def path_case(path, M, T):
    """-> (images, params, unary, G, mus, images compared)"""
    img, sf = helpers.MF64_PATH_CONFIG[path]
    images = helpers.fused_images(img)
    unary, G = inputs(images, M, 200 + M + T)
    return images, grad_params(sf, T), unary, G, None, [1]


def label_case(M, T):
    images = tiny_images(M)
    unary, G = inputs(images, M, 300 + M + T)
    return images, grad_params(1.0, T), unary, G, None, [0, 1]


def set_case(name, mu):
    p = helpers.make_params(helpers.PARAM_SETS[name][0], 3)
    images = helpers.set_images(helpers.PARAM_SETS[name][2], 19, 23, 2)
    M = 6
    unary, G = inputs(images, M, 400)
    return images, p, unary, G, (compat_mats("nonsym", M, 9) if mu == "nonsym" else None), [0, 1]


def configs():
    """Every (name, case) the GPU tests compare with the truth."""
    out = [("path-%s-%d-%d" % (path, M, T), lambda a=(path, M, T): path_case(*a))
           for path in sorted(helpers.MF64_PATH_CONFIG) for M, T in PATH_MT]
    out += [("labels-%d-%d" % (M, T), lambda a=(M, T): label_case(*a))
            for M in LABELS for T in ITERS if label_case_runs(M, T)]
    out += [("set-%s-%s" % (n, mu), lambda a=(n, mu): set_case(*a)) for n in SET_NAMES for mu in SET_MU]
    return out


# the reference's own kernel_grad, frozen for machines without the reference build
GOLDEN_CASES = ("potts_noise", "potts_smooth_sf12", "matrix_noise", "potts_aniso_rgb")


def golden_inputs(name):
    """-> (image (H, W, 3), unary (H, W, M), G, params, mus or None) of one golden case."""
    H, W = 9, 11
    img, sf, M, mu, values = {"potts_noise": ("noise", 1.0, 6, None, None),
                              "potts_smooth_sf12": ("smooth", 12.0, 2, None, None),
                              "matrix_noise": ("noise", 1.0, 6, "sym", None),
                              "potts_aniso_rgb": ("noise", None, 3, None, helpers.PARAM_SETS["aniso_rgb"][0])}[name]
    image = helpers.small_image(np.random.RandomState(3), H, W, img)
    p = helpers.make_params(values, 3) if values is not None else grad_params(sf, 3)
    unary = helpers.log_unary(1, H, W, M, 3, scale=1.0)[0]
    return image, unary, upstream(H, W, M, 4), p, (compat_mats(mu, M, 5) if mu else None)
