"""The case table of test_gpu_label_counts.py reaches what it claims to (no GPU needed): every fused instantiation
MP = 4..32 meets shared-memory tiles, spatial and bilateral direct tiles and hybrid tiles, tail1 and non-tail1 label
counts both occur, and the wide path sees every remainder mod 4.  The tile paths are predicted from the oracle's
lattices with the thresholds of csrc/common.cuh, for an H100 SXM (132 SMs), so a change of images, shapes or
thresholds that hollows out the GPU test fails here."""
import numpy as np
import pytest

import helpers
from helpers import (FUSED_CONFIGS, HYBRID_M, MAX_FUSED, RENORM_M, WIDE_M, fused_images, hybrid_images, padded,
                     predict_tile_paths, tail1)

SMS = 132
ALL_MP = set(range(4, MAX_FUSED + 1, 4))


@pytest.fixture(scope="module")
def fused_paths():
    return {(img, sf): predict_tile_paths(fused_images(img), sf, SMS) for img, sf in FUSED_CONFIGS}


def test_constants_parsed_from_the_sources():
    k = helpers.csrc_constants()
    for name in ("DSRG_MAXLOC_SP", "DSRG_MAXLOC_BI", "DSRG_MAXLOC_HY", "DSRG_HY_MIN_TILES", "DSRG_HY_MIN_COVER"):
        assert k[name] > 0, name
    assert k["kTileW"] * k["kTileH"] == 256
    assert helpers.tile_geometry(321, 321) == (11, 30, 41)   # api.cu: 11 tiles of 30 instead of 10 x 32 + 1
    assert helpers.tile_geometry(41, 45) == (2, 23, 6)


def test_every_fused_instantiation_meets_every_tile_path(fused_paths):
    kinds = {}
    for (img, sf), p in fused_paths.items():
        sp, bi = set(p["sp"]), set(p["bi"].ravel())
        kinds[(img, sf)] = (sp, bi)
    # one configuration per path, all of them run at every M of 1..32
    assert kinds[("smooth", 1.0)] == ({"smem"}, {"smem"})
    assert "direct" in kinds[("noise", 1.0)][1]
    assert "direct" in kinds[("smooth", 12.0)][0]
    assert all(p["hybrid_tiles"] == 0 for p in fused_paths.values())   # small passes stay off the hybrid kernel
    assert {padded(M) for M in range(1, MAX_FUSED + 1)} == ALL_MP


def test_hybrid_cases_cover_every_instantiation():
    image = hybrid_images()
    p = predict_tile_paths(image, 1.0, SMS)
    B = image.shape[0]
    tiles_x, _, tiles_y = helpers.tile_geometry(*image.shape[1:3])
    assert tiles_x * tiles_y * B >= 16 * SMS                      # the pass clears hybrid_tiles_on
    assert p["hybrid_tiles"] >= helpers.csrc_constants()["DSRG_HY_MIN_TILES"] * SMS
    assert all(set(p["bi"][b]) & {"hybrid"} for b in range(B))
    assert {padded(M) for M in HYBRID_M} == ALL_MP
    assert {tail1(M) for M in HYBRID_M} == {True, False}
    assert 24 in HYBRID_M                                         # MP 24 without tail1


def test_tail1_and_full_quads_both_occur():
    assert [M for M in range(1, MAX_FUSED + 1) if tail1(M)] == [1, 5, 9, 13, 17, 21, 25, 29]
    assert {padded(M) for M in helpers.FUSED_ITER_M} == ALL_MP
    assert {tail1(M) for M in helpers.FUSED_ITER_M} == {True, False}


def test_wide_and_renormalisation_cases():
    assert all(M > MAX_FUSED for M in WIDE_M) and max(WIDE_M) == 255
    assert {M % 4 for M in WIDE_M} == {0, 1, 2, 3}
    # numpy_sum: n < 8, one block, the block tail, the split above 128 and the second split from 249 labels on
    assert min(RENORM_M) < 8 and 128 in RENORM_M and 129 in RENORM_M and max(RENORM_M) >= 249
    assert any(M > 128 and (M // 2) % 8 for M in RENORM_M)          # a split point that is rounded down


def test_hybrid_rule_on_hand_made_tiles():
    """_hybrid_cover_ok against tiles.cu's rule worked by hand."""
    k = helpers.csrc_constants()
    npix = 256
    # 256 vertices touched 6 times each: all local (c = 6 fits), full coverage
    assert helpers._hybrid_cover_ok(np.full(256, 6), npix, k)
    # every incidence on its own vertex: c >= 2 keeps nothing
    assert not helpers._hybrid_cover_ok(np.ones(1536, int), npix, k)
    # 300 vertices of 3 and 636 singletons: c = 4 keeps none, c = 3 has 300 > 256 -> threshold 4, extra = 256
    # vertices of count 3 -> 768 of 1536 incidences = 50 %
    counts = np.concatenate([np.full(300, 3), np.ones(636, int)])
    assert counts.sum() == 1536
    assert helpers._hybrid_cover_ok(counts, npix, k) == (768 * 100 >= 1536 * k["DSRG_HY_MIN_COVER"])
