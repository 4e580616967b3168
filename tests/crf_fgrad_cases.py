"""Cases and the per-case bar of the feature-gradient tests (test_crf_fgrad_cpu.py, test_gpu_crf_fgrad.py).

The truth is oracle/crf_fgrad_oracle.feature_grad in float64 on the frozen lattices: dL/df per pixel (N, 5) and
dL/dtheta_gamma (2,).  A case's bar is built like crf_kgrad_cases.KgradTruth's, per feature channel: BAR_K times the
largest error over the pixels of the float32 models (helpers.BAR_MODELS), at least FGRAD_FLOOR times the largest
magnitude of the channel's terms before they cancel.  The device sums a pixel's terms in float32 over its incidences,
labels and iterations, a chain far shorter than 64 adds, so its rounding error is below 2^-18 of that magnitude; the
floor is four times that.

Features: "image" is the image path's own float32(x)/theta_alpha, ..., "random" uniform noise in a box of side 12 (a
lattice as scattered as a noise image's), "guide" a smooth learned-looking embedding: a random 5 x 8 projection of the
image's colours and position.
"""
import numpy as np

import helpers
from crf_compat_cases import compat_mats
from crf_grad_cases import grad_params, upstream
from oracle import crf_fgrad_oracle as F

FGRAD_FLOOR = 2.0 ** -16
FEATURE_KINDS = ("image", "random", "guide")


def features_of(kind, image, params, seed):
    """(H, W, 5) float32 bilateral features of one image."""
    H, W = image.shape[:2]
    if kind == "image":
        return F.image_features(image, params)
    rng = np.random.RandomState(seed)
    if kind == "random":
        return rng.uniform(-6, 6, (H, W, 5)).astype(np.float32)
    y, x = np.mgrid[0:H, 0:W]
    raw = np.concatenate([image.astype(np.float64) / 32.0, x[..., None] / 8.0, y[..., None] / 8.0,
                          np.sin(x / 5.0)[..., None], np.cos(y / 4.0)[..., None], np.ones((H, W, 1))], 2)   # (H, W, 8)
    P = rng.randn(5, 8) * 0.7
    return (raw @ P.T).astype(np.float32)


class FgradTruth(object):
    """float64 dL/df (N, 5) and dL/dtheta_gamma of one image's case, and their bars."""

    def __init__(self, features, params, unary, G, mus=None, models=helpers.BAR_MODELS):
        self.fz = F.Frozen(F.FeatProblem(features, params))
        self.unary, self.G, self.mus = unary, G, mus
        self.want, self.want_sp, mag = F.feature_grad(self.fz, unary, G, mus)
        errs, errs_sp = [np.zeros(5)], [np.zeros(2)]
        for m in models:
            kw = dict(m)
            df, dsp, _ = F.feature_grad(self.fz, unary, G, mus, dtype=np.float32, **kw)
            errs.append(np.abs(df - self.want).max(0))
            errs_sp.append(np.abs(dsp - self.want_sp))
        self.err = np.max(errs, axis=0)
        self.bar = np.maximum(helpers.BAR_K * self.err, FGRAD_FLOOR * mag.max(0))
        self.bar_sp = np.maximum(helpers.BAR_K * np.max(errs_sp, axis=0), FGRAD_FLOOR * np.abs(self.want_sp) + 1e-30)

    def check(self, got, got_sp=None, what=""):
        """got (N, 5) or (5, H, W) as the device writes it."""
        got = np.asarray(got, np.float64)
        if got.shape[0] == 5:
            got = got.reshape(5, -1).T
        assert np.all(np.isfinite(got)), what
        err = np.abs(got - self.want).max(0)
        assert np.all(err <= self.bar), "%s err %s bar %s" % (what, err, self.bar)
        if got_sp is not None:
            e = np.abs(np.asarray(got_sp, np.float64) - self.want_sp)
            assert np.all(e <= self.bar_sp), "%s theta_sp err %s bar %s" % (what, e, self.bar_sp)

    def mutant_excess(self, mutant):
        """max over pixels and channels of |mutant - want| / bar for the float32 restatement with `mutant`."""
        got = F.feature_grad(self.fz, self.unary, self.G, self.mus, mutant=mutant, dtype=np.float32)[0]
        return float((np.abs(got - self.want) / np.maximum(self.bar, 1e-300)).max())


def inputs(B, H, W, M, seed):
    return helpers.log_unary(B, H, W, M, seed, scale=1.0), np.stack([upstream(H, W, M, seed + b) for b in range(B)])


def case(img, sf, kind, M, T, mu=None, H=None, W=None, seed=0):
    """-> (images (B, H, W, 3), features (B, H, W, 5), params, unary, G, mus) of a two-image case; img is one of
    helpers.fused_images' kinds (or "noise" at H x W)."""
    if H is None:
        images = helpers.fused_images(img)
    else:
        images = np.stack([helpers.small_image(np.random.RandomState(seed + 70 + b), H, W, img) for b in range(2)])
    p = grad_params(sf, T)
    feats = np.stack([features_of(kind, images[b], p, seed + b) for b in range(images.shape[0])])
    unary, G = inputs(images.shape[0], images.shape[1], images.shape[2], M, 500 + seed + M + T)
    mus = compat_mats(mu, M, 9) if mu else None
    return images, feats, p, unary, G, mus


# the reference's own FULL_KERNEL kernel_grad, frozen for machines without the reference build
GOLDEN = "crf_fgrad_ref.npz"
GOLDEN_CASES = ("potts_guide", "potts_random", "matrix_guide")


def golden_inputs(name):
    """-> (features (H, W, 5), unary (H, W, M), G, params, mus or None) of one golden case."""
    H, W = 9, 11
    kind, M, mu = {"potts_guide": ("guide", 6, None), "potts_random": ("random", 3, None),
                   "matrix_guide": ("guide", 6, "sym")}[name]
    image = helpers.small_image(np.random.RandomState(3), H, W, "photo")
    p = grad_params(1.0, 3)
    unary = helpers.log_unary(1, H, W, M, 3, scale=1.0)[0]
    return features_of(kind, image, p, 8), unary, upstream(H, W, M, 4), p, (compat_mats(mu, M, 5) if mu else None)
