"""CPU tests of what tests/test_gpu_crf_params.py relies on: the claims of its parameter table (helpers.PARAM_SETS:
non-square images, the tile paths each decoupled set reaches, what the anisotropic and degenerate sets change in the
lattices), the key-range edge of the strip restated per axis (helpers.key_range_ok, api.cu:key_range_ok), the numpy
restatement of k_lattice_insert against the oracle bit for bit at every set, and the generalised helpers giving what
they gave for crf_params(sf)."""
import numpy as np
import pytest

import helpers
from helpers import (KEY_EDGE_B, KEY_EDGE_BI, KEY_EDGE_MAX_KEY, KEY_EDGE_SHAPE, KEY_EDGE_SP, PARAM_SETS, PARAM_TINY,
                     check_restatement, edge_params, key_range_ok, lattice_scales, oracle_lattices, param_set_images,
                     set_images, set_params)
from dsrg_b200 import api

SMS = 132            # an H100 SXM's SMs: the hybrid gate and k_tile_demote's threshold depend on it
down = lambda s: float(np.nextafter(np.float32(s), np.float32(0)))   # noqa: E731


def key_terms(sigma, H, W):
    """The per-feature terms |f_max| * scale of key_range_ok."""
    fmax = [(W - 1) / np.float32(sigma[0]), (H - 1) / np.float32(sigma[1])] + [255.0 / np.float32(s) for s in sigma[2:]]
    return [float(abs(f) * s) for f, s in zip(fmax, lattice_scales(len(sigma)))]


@pytest.mark.parametrize("name", list(PARAM_SETS))
def test_restatement_matches_the_oracle(name):
    """k_lattice_insert restated in float32 gives the oracle's barycentric weights bit for bit, and its vertices, on
    every image of every set (the largest image only once)."""
    images = param_set_images(name)
    params = set_params(name)
    for b in range(min(len(images), 2)):
        keys = check_restatement(images[b], params)
        assert keys[0] <= 32767 and keys[1] <= 2047
    tiny = set_images(PARAM_SETS[name][2], *PARAM_TINY, 1)
    check_restatement(tiny[0], params)


def test_table_claims():
    shapes = {}
    for name, (values, n_iters, kind, (H, W), B, want) in PARAM_SETS.items():
        assert H != W, name
        images = param_set_images(name)
        assert images.shape == (B, H, W, 3), name
        p = set_params(name)
        assert helpers.pairwise_args(p) == tuple(float(np.float32(v)) for v in values)
        pairing = helpers.tile_pairing(helpers.predict_tile_paths(images, p, SMS))
        if want is not None:
            assert pairing == want, (name, pairing)
        shapes[name] = (H, W)
    assert {v for v in (PARAM_SETS[n][5] for n in PARAM_SETS) if v} == \
        {("direct", "smem"), ("smem", "direct"), ("direct", "hybrid")}
    # the inverse anisotropic set runs on the same images, and it changes both lattices
    assert np.array_equal(param_set_images("aniso_xy"), param_set_images("aniso_xy_inv"))
    im = param_set_images("aniso_xy")[0]
    a, b = oracle_lattices(im, set_params("aniso_xy")), oracle_lattices(im, set_params("aniso_xy_inv"))
    for k in (0, 1):
        assert not np.array_equal(a.lattice(k).bary, b.lattice(k).bary), k
    # the per-channel set: one smooth channel, one textured, one constant, and each sigma on its own channel matters
    ch = param_set_images("aniso_rgb")[0].astype(np.float64)
    grad = [np.abs(np.diff(ch[..., c], axis=1)).mean() for c in range(3)]
    assert grad[2] == 0 and 0 < 4 * grad[0] < grad[1]
    p = set_params("aniso_rgb")
    p.theta_beta_r, p.theta_beta_b = p.theta_beta_b, p.theta_beta_r
    assert oracle_lattices(ch.astype(np.uint8), p).lattice(1).M != oracle_lattices(ch.astype(np.uint8),
                                                                                  set_params("aniso_rgb")).lattice(1).M
    # the weights: spatial stronger than bilateral, and a negative one
    w = set_params("weights"), set_params("weights_neg")
    assert w[0].w2 > w[0].w1 > 0 and w[1].w2 < 0
    # the degenerate sets collapse: the x feature to ~0 (and the spatial y one), a colour channel
    base = oracle_lattices(param_set_images("aniso_xy")[0], api.crf_params(1.0))
    dx = oracle_lattices(param_set_images("degenerate_x")[0], set_params("degenerate_x"))
    assert dx.lattice(0).M * 5 < base.lattice(0).M
    assert (W - 1) / np.float32(set_params("degenerate_x").theta_alpha_x) < 0.01
    g_im = param_set_images("degenerate_g")[0]
    dg = oracle_lattices(g_im, set_params("degenerate_g"))
    assert dg.lattice(1).M * 5 < oracle_lattices(g_im, api.crf_params(1.0)).lattice(1).M


def test_key_edge_aniso():
    """On the strip the x terms decide: the edge set passes, one float32 step below on either x axis is refused, and
    the same values with x and y swapped are refused, on the strip and never on its transpose."""
    H, W = KEY_EDGE_SHAPE
    assert W > 20 * H
    for sig in (KEY_EDGE_SP, KEY_EDGE_BI):
        t = key_terms(sig, H, W)
        assert t[0] == max(t) and t[0] > 0.8 * sum(t), t   # the x term sits at the limit
        assert key_range_ok(sig, H, W)
        assert not key_range_ok((down(sig[0]),) + tuple(sig[1:]), H, W)
        swapped = (sig[1], sig[0]) + tuple(sig[2:])
        assert not key_range_ok(swapped, H, W)
        assert key_range_ok(swapped, W, H)           # a restatement that paired W with sigma[1] would flip both
        assert key_range_ok((sig[0], down(sig[1])) + tuple(sig[2:]), H, W)   # y has room
    # the edge images reach keys past 1024 in the bilateral's 12-bit fields, inside both ranges
    images = set_images("binary", H, W, KEY_EDGE_B)
    p = edge_params(KEY_EDGE_SP, KEY_EDGE_BI)
    for b in range(KEY_EDGE_B):
        assert check_restatement(images[b], p) == KEY_EDGE_MAX_KEY
    assert 1024 < KEY_EDGE_MAX_KEY[1] <= 2047 and KEY_EDGE_MAX_KEY[0] <= 32767


def test_generalised_helpers_keep_their_results():
    """crf_params(sf, cf) and a scale factor give the helpers the same nine float32 values as the literal pairwise
    call they used to make (CRF.py:31-32), so every existing case keeps its lattices, tile paths and bars."""
    for sf in (1.0, 3.0, 12.0):
        for cf in (13, 20):
            p = helpers.as_params(sf, cf)
            lit = (10, 80 / sf, 80 / sf, cf, cf, cf, 3, 3 / sf, 3 / sf)
            assert helpers.pairwise_args(p) == tuple(float(np.float32(v)) for v in lit), (sf, cf)
            assert p.n_iters == 10
    for img, sf in helpers.FUSED_CONFIGS:
        images = helpers.fused_images(img)
        a = helpers.predict_tile_paths(images, sf, SMS)
        b = helpers.predict_tile_paths(images, api.crf_params(sf), SMS)
        assert a["hybrid_tiles"] == b["hybrid_tiles"]
        assert np.array_equal(a["sp"], b["sp"]) and np.array_equal(a["bi"], b["bi"])
        assert helpers.bilateral_vertices(images[0], sf) == helpers.bilateral_vertices(images[0], api.crf_params(sf))
        for zero in (None, "w1", "w2"):
            for n in (1, 10):
                old = api.crf_params(sf, maxiter=n)
                if zero:
                    setattr(old, zero, 0.0)
                for new in (helpers.mf64_problem_params(sf, zero, n),
                            helpers.mf64_problem_params(api.crf_params(sf, maxiter=3), zero, n)):
                    assert bytes(new) == bytes(old), (sf, zero, n)
    # a dsrg_crf_params passed in is copied, never changed
    p = api.crf_params(1.0)
    helpers.mf64_problem_params(p, "w1", 2)
    assert p.w1 == 10 and p.n_iters == 10
    assert bytes(edge_params()) == bytes(edge_params(helpers.EDGE_SP, helpers.EDGE_BI))
