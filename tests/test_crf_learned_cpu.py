"""The learned CRF at inference (dsrg_crf_batch_learned_dev, dsrg_predict_mask_batch_learned_dev,
nn.dense_crf_inference and the learned keywords of postprocess.predict_mask_batch_dev / predict_masks_dev) without a
GPU: the float64 identities the GPU tests rely on, the composed oracle of the learned predict_mask, the C symbols and
the refusals that need no device."""
import os
import re

import numpy as np
import pytest

import helpers
from crf_compat_cases import compat_mats
from dsrg_b200 import _lib, api
from oracle import crf_compat_oracle, crf_fgrad_oracle, meanfield64, post_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _case(H, W, img, M, seed, T=10, sf=1.0):
    image = helpers.small_image(np.random.RandomState(seed), H, W, img)
    p = helpers.mf64_problem_params(sf, None, T)
    return image, helpers.log_unary(1, H, W, M, seed)[0], p


@pytest.mark.parametrize("M,T", [(1, 3), (5, 10), (33, 2)])
def test_potts_matrices_are_the_potts_forward(M, T):
    """crf_compat_oracle.run with mu = (-w1 I, -w2 I) is the Potts forward of meanfield64 (the identity the GPU file
    checks the matrix inference by)."""
    image, unary, p = _case(9, 11, "noise", M, 3, T)
    P = meanfield64.Problem(image, p)
    q_c = crf_compat_oracle.run(P, unary, compat_mats("potts", M, 0, p.w1, p.w2), T)[T]
    q_p = P.run(unary, T)[T]
    assert float(np.abs(q_c - q_p).max()) <= 1e-12


@pytest.mark.parametrize("img", ["noise", "smooth"])
def test_image_features_are_the_image_forward(img):
    """The feature forward on the image's own float32 features (x/theta_alpha, y/theta_alpha, rgb/theta_beta) is the
    image forward: the same lattice, so the same marginals."""
    image, unary, p = _case(10, 13, img, 4, 5, 5)
    f = crf_fgrad_oracle.image_features(image, p)
    q_f = crf_fgrad_oracle.FeatProblem(f, p).run(unary, 5)[5]
    q_i = meanfield64.Problem(image, p).run(unary, 5)[5]
    assert float(np.abs(q_f - q_i).max()) <= 1e-12


def learned_crf(mus=None, features=None, n_iters=10):
    """The learned CRF in float64 as post_oracle's CRF step takes it: (im, unary (H, W, M)) -> marginals (H, W, M), with
    matrices mus = (mu_bi, mu_sp) and / or features (H, W, 5) in place of CRF()'s Potts weights and image features."""
    def crf(im, unary):
        p = api.crf_params(1.0, 13, n_iters)
        P = crf_fgrad_oracle.FeatProblem(features, p) if features is not None else meanfield64.Problem(im, p)
        u = np.asarray(unary, np.float32)
        if mus is None:
            return P.run(u, n_iters)[n_iters]
        return crf_compat_oracle.run(P, u, mus, n_iters)[n_iters]
    return crf


def learned_predict_mask(monkeypatch, which, crf, *args):
    """post_oracle.predict_mask_ms / _gt with `crf` in place of CRF(im, log(probs), scale_factor=1.0)."""
    monkeypatch.setattr(post_oracle, "_crf", crf)
    return getattr(post_oracle, which)(*args)


def _margin_agree(a_labels, b_labels, probs, bound=2e-4):
    top2 = np.sort(probs, axis=2)[:, :, -2:]
    sure = (top2[:, :, 1] - top2[:, :, 0]) > bound
    return bool(np.array_equal(a_labels[sure], b_labels[sure]))


@pytest.mark.parametrize("which", ["predict_mask_ms", "predict_mask_gt"])
@pytest.mark.parametrize("kind", ["potts_matrices", "image_features"])
def test_composed_oracle_reproduces_post_oracle_at_the_identities(monkeypatch, which, kind):
    """The learned predict_mask's oracle (post_oracle's steps, the learned CRF in their CRF step) at mu = -w I or at the
    image's own features gives post_oracle's marginals within the CRF bound and its label map wherever the top two
    marginals are 2e-4 apart: what the GPU file's predict_mask identities compare against."""
    M, H, W = 5, 12, 15
    rng = np.random.RandomState(11)
    im = helpers.small_image(rng, H, W, "noise")
    blob = rng.randn(M, 5, 6).astype(np.float32) * 3
    args = (im, [blob, rng.randn(M, 4, 5).astype(np.float32)]) if which == "predict_mask_ms" else (im, blob, [2, 4])
    want_l, want_p = getattr(post_oracle, which)(*args)
    p = api.crf_params(1.0)
    if kind == "potts_matrices":
        crf = learned_crf(mus=compat_mats("potts", M, 0, p.w1, p.w2))
    else:
        crf = learned_crf(features=crf_fgrad_oracle.image_features(im, p))
    got_l, got_p = learned_predict_mask(monkeypatch, which, crf, *args)
    assert float(np.abs(got_p - want_p).max()) <= 1e-4
    assert _margin_agree(got_l, want_l, want_p)


def test_new_symbols_are_declared_and_exported():
    header = open(os.path.join(ROOT, "include", "dsrg_b200.h")).read()
    L = _lib.lib()
    for name in ("dsrg_crf_batch_learned_dev", "dsrg_predict_mask_batch_learned_dev"):
        assert re.search(r"\bint %s\(" % name, header), name
        assert name in _lib.SIGNATURES
        getattr(L, name)   # AttributeError when the library does not export it
    assert L.dsrg_version() >= 117


def _torch():
    return pytest.importorskip("torch")


def test_dense_crf_inference_refusals_without_gpu():
    torch = _torch()
    from dsrg_b200 import nn
    u = torch.zeros(1, 3, 4, 5)
    img = torch.zeros(1, 4, 5, 3, dtype=torch.uint8)
    f = torch.zeros(1, 5, 4, 5)
    with pytest.raises(ValueError, match="image is not used"):
        nn.dense_crf_inference(u, img, features_bi=f)
    with pytest.raises(ValueError, match="image must be"):
        nn.dense_crf_inference(u, None)
    with pytest.raises(ValueError, match="at most|1 <= M"):
        nn.dense_crf_inference(torch.zeros(1, 256, 4, 5), img)
    with pytest.raises(ValueError, match="maxiter"):
        nn.dense_crf_inference(u, img, maxiter=-1)
    with pytest.raises(ValueError, match="CUDA tensor"):
        nn.dense_crf_inference(u, img)


def test_predict_mask_batch_dev_learned_needs_smooth():
    torch = _torch()
    from dsrg_b200 import postprocess
    with pytest.raises(ValueError, match="smooth=True"):
        postprocess.predict_mask_batch_dev(torch.zeros(1, 4, 5, 3, dtype=torch.uint8), [torch.zeros(1, 3, 2, 2)],
                                           smooth=False, compat_bi=torch.zeros(3, 3))
