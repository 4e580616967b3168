"""Cases and bars of the kernel-bandwidth and feature gradients above 32 labels (test_crf_wide_kgrad_cpu.py,
test_gpu_crf_wide_kgrad.py).

The truths are oracle/crf_kgrad_oracle.theta_grad and oracle/crf_fgrad_oracle.feature_grad in float64 on the frozen
lattices.  The float32-model part of a bar is crf_kgrad_cases.KgradTruth's / crf_fgrad_cases.FgradTruth's: BAR_K
times the largest error of helpers.BAR_MODELS, each run forward and backward in float32.  The floor is re-derived for
the label-chunked kernel, whose sums are deeper than the fused path's:

- k_wide_kg_pass forms s_r at an incidence as one fma chain over the label quads in ascending order, 8 terms per quad
  (x . Vy and u . Vg): 8 ceil(M/4) terms, 72 at 33 labels, 168 at 81 and 512 at 255.
- Then, as on the fused path: the pixel's incidences (at most 6) in kg_features, a warp's tree (5), the block's 8
  warps, the iterations and the normalisation term added to the block's sums (at most 11), and the blocks of the
  image in order (at most 7 for the 41x41 cases held to the truth): 37 more, below 64.

So a sum has depth below 8 ceil(M/4) + 64, and its float32 rounding error is below (8 ceil(M/4) + 64) 2^-24 of the
sum of the magnitudes of its terms (the oracle's A).  The floor is four times that: 2^-14.9 of A at 33 labels, 2^-13.7
at 81 and 2^-12.8 at 255, where the narrow KGRAD_FLOOR (2^-16) assumes a depth below 64 and does not carry over.  A
pixel's dL/df is the same chain without the warp, block and image sums; it gets the same floor (FgradTruth's per-channel
magnitude).  dL/dtheta_gamma of the feature pass is an image sum like the theta path's: its floor is the same times
the sum over the pixels of |f_i| times the magnitude of (dL/df)_i's terms, crf_kgrad_oracle.theta_grad's A for the
spatial lattice (SpatialView).  A floor relative to the value, as FgradTruth's, sits below that rounding wherever the
sum cancels, and it does cancel: a kernel does not change when a feature channel is shifted, so sum_i (dL/df)_i is zero
and A exceeds |dL/dtheta_gamma| thousandfold.

CONFIGS are the cases the GPU file compares with the truth, so that the CPU file can show every oracle mutant outside
the bars the device is held to.
"""
import math

import numpy as np

import helpers
from crf_compat_cases import compat_mats
from crf_fgrad_cases import FgradTruth, features_of
from crf_grad_cases import grad_params, upstream
from crf_kgrad_cases import KgradTruth
from oracle import crf_fgrad_oracle as F
from oracle import crf_kgrad_oracle as K

WIDE_M = (33, 36, 81, 128, 255)   # phantom lanes in the last quad (3, 1) and whole quads
ITERS = (0, 1, 2, 10)
GOLDEN = "crf_wide_kgrad_ref.npz"


def wide_floor(M):
    """The bar's floor relative to the magnitude of the terms at M labels (the module docstring)."""
    return 4.0 * (8 * math.ceil(M / 4.0) + 64) * 2.0 ** -24


class WideKgradTruth(KgradTruth):
    """KgradTruth with the label-chunked kernel's floor."""

    def __init__(self, image, params, unary, G, mus=None, models=helpers.BAR_MODELS):
        KgradTruth.__init__(self, image, params, unary, G, mus, models)
        self.bar = np.maximum(helpers.BAR_K * self.err, wide_floor(unary.shape[-1]) * self.A / self.th)


class SpatialView(object):
    """A feature problem (crf_fgrad_oracle.Frozen) seen as crf_kgrad_oracle.theta_grad sees an image's: the spatial
    lattice at the problem's theta_gamma, the bilateral one at the given features.  theta_grad on it gives the spatial
    dL/dtheta_gamma (entries 5, 6) and A, the magnitude of its terms."""

    def __init__(self, fz):
        self.fz, self.problem, self.rank = fz, fz.problem, [fz.sp_rank, fz.rank]
        self.theta0 = np.concatenate([np.ones(5), fz.theta_sp])   # the bilateral entries are not used

    def frozen_problem(self, theta):
        return self.fz.frozen_problem(self.fz.f32.astype(np.float64))

    def features(self, k, theta):
        return self.fz.sp_f if k == 0 else self.fz.f32.astype(np.float64)


class WideFgradTruth(FgradTruth):
    """FgradTruth with the label-chunked kernel's floors: per pixel relative to the magnitude of the terms of dL/df,
    and for dL/dtheta_gamma relative to A over the spatial lattice (the module docstring)."""

    def __init__(self, features, params, unary, G, mus=None, models=helpers.BAR_MODELS):
        FgradTruth.__init__(self, features, params, unary, G, mus, models)
        fl = wide_floor(unary.shape[-1])
        mag = F.feature_grad(self.fz, unary, G, mus)[2]   # the magnitude of each pixel's terms, as FgradTruth's
        self.bar = np.maximum(self.bar, fl * mag.max(0))
        view = SpatialView(self.fz)
        dth, _, A = K.theta_grad(view, view.theta0, unary, G, int(params.n_iters), mus)
        assert np.allclose(dth[5:7], self.want_sp, rtol=1e-12, atol=0), (dth[5:7], self.want_sp)
        self.bar_sp = np.maximum(self.bar_sp, fl * A[5:7] / self.fz.theta_sp)


def inputs(B, H, W, M, seed):
    return helpers.log_unary(B, H, W, M, seed, scale=1.0), np.stack([upstream(H, W, M, seed + b) for b in range(B)])


def images_of(img, H, W, seed, B=2):
    return np.stack([helpers.small_image(np.random.RandomState(seed + 70 + b), H, W, img) for b in range(B)])


def label_case(M, T, sf):
    """-> (images, params, unary, G, mus): two noise images of 13 x 17 (phantom lanes) at M labels, T iterations."""
    images = images_of("noise", 13, 17, M + T)
    unary, G = inputs(2, 13, 17, M, 800 + M + T)
    return images, grad_params(sf, T), unary, G, None


def image_case(img, mu, T=3):
    """81 labels on 41 x 41 smooth / photo / noise images; mu: "potts_host", "potts_dev" or "nonsym"."""
    images = images_of(img, 41, 41, 5)
    unary, G = inputs(2, 41, 41, 81, 900)
    return images, grad_params(12.0, T), unary, G, (compat_mats("nonsym", 81, 9) if mu == "nonsym" else None)


def aniso_case(name, mu):
    p = helpers.make_params(helpers.PARAM_SETS[name][0], 3)
    images = helpers.set_images(helpers.PARAM_SETS[name][2], 19, 23, 2)
    unary, G = inputs(2, 19, 23, 36, 950)
    return images, p, unary, G, (compat_mats("nonsym", 36, 9) if mu == "nonsym" else None)


def feature_case(kind, M, T, mu=None):
    """-> (images, features (B, H, W, 5), params, unary, G, mus) on two photo-like 23 x 29 images."""
    images = images_of("photo", 23, 29, 3)
    p = grad_params(1.0, T)
    feats = np.stack([features_of(kind, images[b], p, 11 + b) for b in range(2)])
    unary, G = inputs(2, 23, 29, M, 1000 + M + T)
    return images, feats, p, unary, G, (compat_mats(mu, M, 9) if mu else None)


LABEL_RUNS = [(M, T, sf) for M in WIDE_M for T in ITERS for sf in (1.0, 12.0) if T < 10 or M in (33, 81)]
IMAGE_RUNS = [(img, mu) for img in ("smooth", "photo", "noise") for mu in ("potts_host", "potts_dev", "nonsym")]
ANISO_RUNS = [(n, mu) for n in ("aniso_xy", "aniso_rgb") for mu in ("potts", "nonsym")]
FEATURE_RUNS = [(kind, M, T, mu) for kind in ("image", "guide", "random") for M, T in ((33, 2), (81, 3), (255, 1))
                for mu in (None, "nonsym")] + [("guide", 81, 10, None), ("guide", 81, 0, None)]


def configs():
    """Every (name, case thunk, "theta" or "feat") the GPU file compares with the truth."""
    out = [("labels-%d-%d-%g" % a, lambda a=a: label_case(*a), "theta") for a in LABEL_RUNS]
    out += [("image-%s-%s" % a, lambda a=a: image_case(*a), "theta") for a in IMAGE_RUNS]
    out += [("aniso-%s-%s" % a, lambda a=a: aniso_case(*a), "theta") for a in ANISO_RUNS]
    out += [("feat-%s-%d-%d-%s" % a, lambda a=a: feature_case(*a), "feat") for a in FEATURE_RUNS]
    return out


# the reference's own kernel_grad above 32 labels, frozen for machines without the reference build:
# name -> (H, W, image, M, scale factor, T, seed, None / "sym", "theta" or "feat")
GOLDEN_CASES = {
    "theta_potts_33": (9, 11, "noise", 33, 1.0, 3, 3, None, "theta"),
    "theta_sym_81": (9, 11, "smooth", 81, 12.0, 2, 5, "sym", "theta"),
    "feat_potts_81": (9, 11, "photo", 81, 1.0, 2, 7, None, "feat"),
    "feat_sym_33": (9, 11, "photo", 33, 1.0, 3, 9, "sym", "feat"),
}


def golden_inputs(name):
    """-> (image (H, W, 3), features (H, W, 5) or None, unary (H, W, M), G, params, mus or None, kind)."""
    H, W, img, M, sf, T, seed, mu, kind = GOLDEN_CASES[name]
    image = helpers.small_image(np.random.RandomState(seed), H, W, img)
    p = grad_params(sf, T)
    feats = features_of("guide", image, p, seed + 1) if kind == "feat" else None
    unary = helpers.log_unary(1, H, W, M, seed, scale=1.0)[0]
    return image, feats, unary, upstream(H, W, M, seed + 2), p, (compat_mats(mu, M, seed) if mu else None), kind
