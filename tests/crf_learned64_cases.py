"""Cases, the float64 truth and the bar of the learned-CRF inference tests (test_gpu_crf_learned64.py, checked on the
CPU by test_crf_learned64_cpu.py): compatibility matrices and caller-given bilateral features through
Engine.crf_learned_dev, nn.dense_crf_inference and the learned predict_mask, at every padded label width of the fused
kernels and on the label-chunked path.

The truth is oracle/crf_compat_oracle.run in float64 (meanfield64.Problem.run when the case has no matrices), on the
image's lattices (meanfield64.Problem) or on the features' (crf_fgrad_oracle.FeatProblem).  A case's bar is built as
helpers.mf64_truth_and_bar builds it: helpers.BAR_K times the largest error of the float32 models of
helpers.BAR_MODELS (the device's operation order included), at least helpers.BAR_FLOOR, per image and per n.

No case sits at an identity of the Potts CRF: the matrices are not symmetric and the features are the image's own
scaled by LEARNED_FEAT_SCALE and shifted by LEARNED_FEAT_SHIFT, so a kernel that dropped, transposed or swapped the
matrices or read the image's features would land outside the bar."""
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import threadpoolctl

import helpers
from crf_compat_cases import compat_mats
from oracle import crf_compat_oracle, crf_fgrad_oracle, meanfield64, post_oracle

# one M per padded width MP = 4, 8, ..., 32: 1, 9 and 25 are tail1 (one real label in the last quad), 6 and 18 have
# two phantom lanes, 16, 24 and 32 none
LEARNED_M = [1, 6, 9, 16, 18, 24, 25, 32]
# the label-chunked path: 33 and 81 leave three phantom lanes in the last quad, 255 one, 36 and 128 none
LEARNED_WIDE_M = [33, 36, 81, 128, 255]
LEARNED_ITERS = (0, 1, 2, 3, 10)
LEARNED_WIDE_ITERS = (0, 1, 2, 10)
# the training forward and backward at the widths COMPAT_M leaves out (MP 12, 16, 20, 28)
LEARNED_TRAIN_M = [9, 16, 18, 25]
LEARNED_FEAT_SCALE, LEARNED_FEAT_SHIFT = 0.8, 3.0

# kind -> (matrices, features): "mats" non-symmetric mu on the image's lattices; "feats" the Potts weights on scaled,
# shifted features; "both"; "sp_only" / "bi_only" the non-symmetric mu of one lattice with the other's mu zero, so a
# failure names the lattice
KINDS = ("mats", "feats", "both", "sp_only", "bi_only")


def learned_features(image, params):
    """(H, W, 5) float32: the image's own bilateral features, scaled and shifted."""
    f = crf_fgrad_oracle.image_features(image, params)
    return (f * np.float32(LEARNED_FEAT_SCALE) + np.float32(LEARNED_FEAT_SHIFT)).astype(np.float32)


def kind_mats(kind, M, seed):
    """(mu_bi, mu_sp) of a kind, or None for the Potts weights."""
    if kind == "feats":
        return None
    mu_bi, mu_sp = compat_mats("nonsym", M, seed)
    if kind == "sp_only":
        mu_bi = np.zeros_like(mu_bi)
    elif kind == "bi_only":
        mu_sp = np.zeros_like(mu_sp)
    return mu_bi, mu_sp


def kind_uses_features(kind):
    return kind in ("feats", "both")


def problem_for(kind, image, params):
    """The float64 restatement's lattices of one (H, W, 3) image under a kind: the scaled features' for "feats" and
    "both", the image's otherwise."""
    if kind_uses_features(kind):
        return crf_fgrad_oracle.FeatProblem(learned_features(image, params), params)
    return meanfield64.Problem(image, params)


def run_learned(problem, unary, mus, n_iters, **kw):
    """Q_0..Q_n of the learned CRF: crf_compat_oracle.run with matrices, the problem's Potts forward without."""
    if mus is None:
        return problem.run(unary, n_iters, **kw)
    return crf_compat_oracle.run(problem, unary, mus, n_iters, **kw)


class LearnedTruth(object):
    """The float64 marginals of one image's learned CRF after every n of `iters` (q64[n]) and their bars (bar[n]);
    spread[n] is the largest float32 model error.  problem: a meanfield64.Problem or a crf_fgrad_oracle.FeatProblem;
    mus = (mu_bi, mu_sp) or None (the problem's Potts weights).  Forward only."""

    def __init__(self, problem, unary, mus, iters=LEARNED_ITERS):
        self.iters = tuple(iters)
        T = max(self.iters)
        jobs = [dict(dtype=np.float64)] + [dict(dtype=np.float32, **m) for m in helpers.BAR_MODELS]
        for j in jobs:                      # the norms are cached on the problem: fill the cache before the threads
            problem.norms(j["dtype"], j.get("splat_order"))
        # the matrix products of the oracle's float32 models go through BLAS; concurrent calls into a multi-threaded
        # OpenBLAS from these threads have returned wrong products, so BLAS runs single-threaded here
        with threadpoolctl.threadpool_limits(1, user_api="blas"), \
                ThreadPoolExecutor(min(len(jobs), os.cpu_count() or 1)) as ex:
            runs = list(ex.map(lambda kw: run_learned(problem, unary, mus, T, **kw), jobs))
        self.q64 = {n: runs[0][n] for n in self.iters}
        self.spread = {n: max(float(np.abs(r[n] - self.q64[n]).max()) for r in runs[1:]) for n in self.iters}
        self.bar = {n: max(helpers.BAR_K * self.spread[n], helpers.BAR_FLOOR) for n in self.iters}
        assert max(self.spread.values()) < 1e-3, "the float32 models are not float32 noise: %r" % self.spread


def feature_tile_kinds(features, H, W, hybrid_on):
    """helpers.lattice_tile_kinds of the bilateral lattice built on (H, W, 5) features."""
    from oracle import crf_oracle
    lat = crf_oracle.OracleLattice(np.ascontiguousarray(features, np.float32).reshape(H * W, 5))
    return helpers.lattice_tile_kinds(lat.offset, H, W, 1, hybrid_on)


def predicted_paths(image, params, kind, sms):
    """helpers.predict_tile_paths, with the bilateral tiles of a feature kind predicted from its features."""
    pred = helpers.predict_tile_paths(image, params, sms)
    if kind_uses_features(kind):
        B, H, W = image.shape[:3]
        gate = helpers.hybrid_tiles_on(H, W, B, sms)
        pred["bi"] = np.stack([feature_tile_kinds(learned_features(image[b], params), H, W, gate) for b in range(B)])
        pred["hybrid_tiles"] = helpers.demote_hybrid_tiles(pred["bi"], sms)
    return pred


def reaches(pred, path):
    sp, bi = helpers.tile_pairing(pred)
    return {"smem": (sp, bi) == ("smem", "smem"), "bi_direct": bi == "direct", "sp_direct": sp == "direct"}[path]


# ---- the learned predict_mask against the composed float64 oracle ----
# kind -> what the learned CRF takes in place of CRF()'s: "mats" non-symmetric mu, "feats" scaled features, "both",
# "theta" other bandwidths with other Potts weights (read on the host)
POST_KINDS = ("mats", "feats", "both", "theta")
POST_THETA_BI, POST_THETA_SP = (60.0, 95.0, 9.0, 16.0, 11.0), (2.0, 4.5)
POST_W1, POST_W2 = 6.5, 1.5
POST_SHAPE, POST_B, POST_M = (47, 61), 3, (21, 81)
POST_SCORE_SHAPES = ((9, 11), (13, 15))             # the scales of "ms"; "gt" takes the first
POST_HYBRID_M, POST_HYBRID_SCORES = 21, (41, 41)
POST_SEED = 40


def post_params(kind):
    """The dsrg_crf_params the learned CRF of a predict_mask kind runs with (absolute sigmas, ten iterations)."""
    from dsrg_b200 import api
    p = api.crf_params(1.0)
    if kind == "theta":
        (p.theta_alpha_x, p.theta_alpha_y, p.theta_beta_r, p.theta_beta_g, p.theta_beta_b) = POST_THETA_BI
        p.theta_gamma_x, p.theta_gamma_y = POST_THETA_SP
        p.w1, p.w2 = POST_W1, POST_W2
    return p


def post_mats(kind, M):
    return compat_mats("nonsym", M, 7) if kind in ("mats", "both") else None


def post_inputs(B, H, W, M, seed, score_shapes=POST_SCORE_SHAPES):
    """images (B, H, W, 3) uint8 photos, scores [(B, M, h, w) float32] per scale and tags (B, M) 0/1."""
    rng = np.random.RandomState(seed)
    images = np.stack([helpers.small_image(rng, H, W, "photo") for _ in range(B)])
    scores = [(rng.randn(B, M, h, w) * 3).astype(np.float32) for h, w in score_shapes]
    tags = (rng.rand(B, M) > 0.7).astype(np.float32)
    return images, scores, tags


def tag_ids(tags_row):
    """post_oracle.predict_mask_gt's labels (1-based class ids without background) of one image's 0/1 tags."""
    return [int(c) for c in np.nonzero(np.asarray(tags_row) > 0.5)[0] if c > 0]


def learned_crf(mus=None, features=None, n_iters=10, params=None):
    """The learned CRF in float64 as post_oracle's CRF step takes it: (im, unary (H, W, M)) -> marginals (H, W, M), with
    matrices mus = (mu_bi, mu_sp) and / or features (H, W, 5) in place of CRF()'s Potts weights and image features;
    params (default CRF()'s api.crf_params(1.0)) gives the sigmas and the Potts weights."""
    def crf(im, unary):
        from dsrg_b200 import api
        p = helpers.as_params(params) if params is not None else api.crf_params(1.0, 13, n_iters)
        p.n_iters = n_iters
        P = crf_fgrad_oracle.FeatProblem(features, p) if features is not None else meanfield64.Problem(im, p)
        return run_learned(P, np.asarray(unary, np.float32), mus, n_iters)[n_iters]
    return crf


def learned_predict_mask(monkeypatch, which, crf, *args):
    """post_oracle.predict_mask_ms / _gt with `crf` in place of CRF(im, log(probs), scale_factor=1.0)."""
    monkeypatch.setattr(post_oracle, "_crf", crf)
    return getattr(post_oracle, which)(*args)


def post_oracle_case(monkeypatch, kind, mode, image, scores_b, tags_row, M):
    """(labels (H, W), marginals (H, W, M)) of one image under a predict_mask kind: scores_b the image's (M, h, w)
    score map of each scale."""
    p = post_params(kind)
    feats = learned_features(image, p) if kind in ("feats", "both") else None
    crf = learned_crf(post_mats(kind, M), feats, 10, p)
    if mode == "ms":
        return learned_predict_mask(monkeypatch, "predict_mask_ms", crf, image, list(scores_b))
    return learned_predict_mask(monkeypatch, "predict_mask_gt", crf, image, scores_b[0], tag_ids(tags_row))


def sure(probs, bound=2e-4):
    """Pixels whose top two marginals are more than `bound` apart: there the label map is decided."""
    top2 = np.sort(probs, axis=-1)[..., -2:]
    return (top2[..., 1] - top2[..., 0]) > bound
