"""test_gpu_crf_learned64.py's cases and bars without a GPU: the float64 restatements agree with each other at the
identities, the bars are tight enough that a transposed, swapped or dropped matrix and the unscaled features land
outside them, the label lists cover every padded width, the tile paths the GPU file claims are reached, and the
learned predict_mask cases are not the Potts CRF in disguise."""
import numpy as np
import pytest

import helpers
from crf_compat_cases import compat_mats
from crf_learned64_cases import (LEARNED_ITERS, LEARNED_M, LEARNED_TRAIN_M, LEARNED_WIDE_ITERS, LEARNED_WIDE_M,
                                 POST_KINDS, POST_SEED, POST_SHAPE, LearnedTruth, kind_mats, post_inputs,
                                 post_oracle_case, predicted_paths, problem_for, reaches, run_learned, sure, tag_ids)
from oracle import crf_fgrad_oracle, meanfield64, post_oracle

H100_SMS = 132


def _image(H, W, img, seed):
    return helpers.small_image(np.random.RandomState(seed), H, W, img)


# ---- the restatements agree with each other ----
@pytest.mark.parametrize("M", [1, 9, 33])
def test_truth_at_potts_matrices_is_meanfield64(M):
    image = _image(9, 11, "noise", 3)
    p = helpers.mf64_problem_params(1.0)
    P = meanfield64.Problem(image, p)
    unary = helpers.log_unary(1, 9, 11, M, 3)[0]
    t = LearnedTruth(P, unary, compat_mats("potts", M, 0, p.w1, p.w2))
    q = P.run(unary, max(LEARNED_ITERS))
    for n in LEARNED_ITERS:
        assert float(np.abs(t.q64[n] - q[n]).max()) <= 1e-12, n


@pytest.mark.parametrize("with_mats", [False, True])
def test_own_features_are_the_image_problem(with_mats):
    """A FeatProblem on the image's own features is the image's Problem, with the Potts weights and with matrices."""
    image = _image(10, 13, "smooth", 5)
    p = helpers.mf64_problem_params(1.0)
    M = 6
    unary = helpers.log_unary(1, 10, 13, M, 5)[0]
    mus = compat_mats("nonsym", M, 2) if with_mats else None
    q_f = run_learned(crf_fgrad_oracle.FeatProblem(crf_fgrad_oracle.image_features(image, p), p), unary, mus, 10)
    q_i = run_learned(meanfield64.Problem(image, p), unary, mus, 10)
    for n in range(11):
        assert float(np.abs(q_f[n] - q_i[n]).max()) <= 1e-12, n


# ---- the bars discriminate ----
def _mutants(kind, mus, image, params):
    """name -> (problem, mus) of the mutant runs of a case."""
    out = {}
    if mus is not None:
        P = problem_for(kind, image, params)
        mu_bi, mu_sp = mus
        out["mu transposed"] = (P, (mu_bi.T, mu_sp.T))
        out["mu_bi and mu_sp swapped"] = (P, (mu_sp, mu_bi))
        out["spatial message dropped"] = (P, (mu_bi, np.zeros_like(mu_sp)))
        out["bilateral message dropped"] = (P, (np.zeros_like(mu_bi), mu_sp))
    if kind in ("feats", "both"):
        out["unscaled features"] = (crf_fgrad_oracle.FeatProblem(crf_fgrad_oracle.image_features(image, params),
                                                                 params), mus)
    return out


# (path or "wide", kind, M): cases of the GPU file, at widths old and new
DISCRIMINATE = [(path, kind, M) for path in sorted(helpers.MF64_PATH_CONFIG) for kind in ("mats", "feats", "both")
                for M in (6, 16, 25)] + [("wide", kind, M) for kind in ("mats", "both") for M in (33, 81)]


@pytest.mark.parametrize("path,kind,M", DISCRIMINATE)
def test_mutants_land_outside_the_bar(path, kind, M):
    if path == "wide":
        image = helpers.wide_images("noise")
        seed, scale, iters = 800 + M, 4.0, LEARNED_WIDE_ITERS
        params = helpers.mf64_problem_params(1.0)
    else:
        img, sf = helpers.MF64_PATH_CONFIG[path]
        image = helpers.fused_images(img)
        seed, scale, iters = 200 + M, 2.0, LEARNED_ITERS
        params = helpers.mf64_problem_params(sf)
    B, H, W = image.shape[:3]
    unary = helpers.log_unary(B, H, W, M, seed=seed, scale=scale)[0]
    mus = kind_mats(kind, M, M)
    truth = LearnedTruth(problem_for(kind, image[0], params), unary, mus, iters)
    T = max(iters)
    for name, (P, m) in _mutants(kind, mus, image[0], params).items():
        q = run_learned(P, unary, m, T, dtype=np.float32)
        ratio = max(float(np.abs(q[n] - truth.q64[n]).max()) / truth.bar[n] for n in iters if n >= 1)
        print("%s %s M%d %s: largest error / bar %.1f" % (path, kind, M, name, ratio))
        assert ratio > 1, name


# ---- coverage ----
def test_label_lists_cover_every_width():
    assert {helpers.padded(M) for M in LEARNED_M} == set(range(4, 33, 4))
    assert all(M <= helpers.MAX_FUSED for M in LEARNED_M)
    assert any(helpers.tail1(M) for M in LEARNED_M) and any(helpers.padded(M) - M == 2 for M in LEARNED_M)
    assert {helpers.padded(M) for M in LEARNED_TRAIN_M} == {12, 16, 20, 28}
    phantoms = {helpers.padded(M) - M for M in LEARNED_WIDE_M}
    assert min(LEARNED_WIDE_M) > helpers.MAX_FUSED and max(LEARNED_WIDE_M) == 255
    assert {0, 1, 3} <= phantoms
    assert {0, 1, 2, 3, 10} <= set(LEARNED_ITERS) and {0, 10} <= set(LEARNED_WIDE_ITERS)


@pytest.mark.parametrize("kind", ["mats", "feats", "both"])
@pytest.mark.parametrize("path", sorted(helpers.MF64_PATH_CONFIG))
def test_fused_cases_reach_their_path(path, kind):
    img, sf = helpers.MF64_PATH_CONFIG[path]
    image = helpers.fused_images(img)
    assert reaches(predicted_paths(image, helpers.mf64_problem_params(sf), kind, H100_SMS), path)


def test_hybrid_cases_reach_hybrid_tiles():
    image = helpers.hybrid_images()
    params = helpers.mf64_problem_params(1.0)
    assert helpers.predict_tile_paths(image, params, H100_SMS)["hybrid_tiles"] > 0
    assert predicted_paths(image, params, "feats", H100_SMS)["hybrid_tiles"] > 0
    assert not helpers.hybrid_tiles_on(*image.shape[1:3], 3, H100_SMS)     # the B = 3 pass of the same engine


# ---- the predict_mask cases are not identities in disguise ----
@pytest.mark.parametrize("mode", ["ms", "gt"])
@pytest.mark.parametrize("kind", POST_KINDS)
def test_predict_mask_cases_change_the_label_map(monkeypatch, kind, mode):
    """Each learned kind changes the label map of CRF()'s predict_mask on at least 1% of the pixels where both are
    sure, so a pass that ignored the matrices, the features or the sigmas would fail the GPU file."""
    M = 21
    H, W = POST_SHAPE
    image, scores, tags = post_inputs(1, H, W, M, POST_SEED + M)
    sc = [s[0] for s in scores] if mode == "ms" else [scores[0][0]]
    got_l, got_p = post_oracle_case(monkeypatch, kind, mode, image[0], sc, tags[0], M)
    monkeypatch.undo()
    if mode == "ms":
        want_l, want_p = post_oracle.predict_mask_ms(image[0], sc)
    else:
        want_l, want_p = post_oracle.predict_mask_gt(image[0], sc[0], tag_ids(tags[0]))
    both = sure(got_p) & sure(want_p)
    frac = float((got_l[both] != want_l[both]).mean())
    print("%s %s: %.1f%% of the sure pixels change" % (kind, mode, 100 * frac))
    assert frac >= 0.01

