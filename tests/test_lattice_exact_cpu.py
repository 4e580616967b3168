"""CPU tests of what tests/test_gpu_lattice_exact.py relies on: the numpy restatement of k_lattice_insert's arithmetic
(helpers.lattice_insert) and of api.cu:key_range_ok, the claims of its case table (phantom lanes, tile widths, the
sigmas at the edge of the key range and the largest |key| they reach), and the bound on the renumbering key that
dsrg_engine_create enforces."""
import os
import re

import numpy as np
import pytest

import helpers
from conftest import ROOT
from helpers import (EDGE_B, EDGE_BI, EDGE_MAX_KEY, EDGE_SHAPE, EDGE_SP, EXACT_BENCH, EXACT_CASES, K_NO_KEY,
                     RENUM_MAX_H_W1, check_restatement, edge_params, exact_images, key_range_ok, lattice_sigmas,
                     phantom_lanes, renum_key_limit, tile_geometry)
from dsrg_b200 import _lib, api


@pytest.mark.parametrize("kind,sf", [("photo", 1.0), ("noise", 12.0), ("binary", 1.0)])
def test_restatement_matches_the_oracle(kind, sf):
    H, W = 21, 33
    image = exact_images(kind, H, W, 1)[0]
    check_restatement(image, api.crf_params(sf, maxiter=1))


def test_edge_sigmas_are_the_edge():
    H, W = EDGE_SHAPE
    down = lambda s: float(np.nextafter(np.float32(s), np.float32(0)))   # noqa: E731
    assert key_range_ok(EDGE_SP, H, W) and key_range_ok(EDGE_BI, H, W)
    assert not key_range_ok((down(EDGE_SP[0]), EDGE_SP[1]), H, W)
    assert not key_range_ok((EDGE_SP[0], down(EDGE_SP[1])), H, W)
    assert not key_range_ok((down(EDGE_BI[0]),) + EDGE_BI[1:], H, W)
    # the bench's own sigmas are far from it
    p = api.crf_params(1.0)
    assert key_range_ok(lattice_sigmas(p, 0), 513, 513) and key_range_ok(lattice_sigmas(p, 1), 513, 513)


def test_bound_holds_on_the_worst_case_images():
    """At the edge sigmas, on images of colours 0 and 255 with every colour corner at the image's corners: the
    restated keys stay inside the packed range, reach EDGE_MAX_KEY (past 1024 in the 12-bit fields, so their top bits
    and sign extension are used), and the restatement is the oracle's."""
    H, W = EDGE_SHAPE
    images = exact_images("binary", H, W, EDGE_B)
    assert {tuple(images[0, y, x]) for y in (0, H - 1) for x in list(range(8)) + list(range(W - 8, W))} == \
        {(r, g, b) for r in (0, 255) for g in (0, 255) for b in (0, 255)}
    for b in range(EDGE_B):
        got = check_restatement(images[b], edge_params())
        assert got == EDGE_MAX_KEY, got
    assert EDGE_MAX_KEY[1] > 1024 and EDGE_MAX_KEY[1] <= 2047 and EDGE_MAX_KEY[0] <= 32767
    # the host bound is conservative on other shapes and sigmas as well
    rng = np.random.RandomState(3)
    for Hh, Ww in ((1, 40), (40, 1), (17, 64)):
        im = helpers.extreme_image(rng, Hh, Ww)
        for scale in (1.0, 1.5, 4.0):
            sig = [s * scale for s in EDGE_BI]
            sig[0] = EDGE_BI[0] * (Ww - 1) / (W - 1) * scale if Ww > 1 else 1.0
            sig[1] = EDGE_BI[1] * (Hh - 1) / (H - 1) * scale if Hh > 1 else 1.0
            if key_range_ok(sig, Hh, Ww):
                assert helpers.max_abs_key(im, sig) <= 2047


def test_case_table():
    for name, (H, W, B, kind, sf, M, P, tile_w) in EXACT_CASES.items():
        assert phantom_lanes(H * W) == P, name
        assert tile_geometry(H, W)[1] == tile_w, name
    table = list(EXACT_CASES.values()) + [EXACT_BENCH + ("", 1.0, 21, phantom_lanes(321 * 321), 30)]
    assert tile_geometry(321, 321)[1] == 30
    assert {c[6] for c in table} == {0, 1, 2, 3}                        # 3, 2 and 1 phantom lanes, and none
    assert {17, 30} <= {c[7] for c in table}
    assert any(c[0] % 8 for c in table)
    shapes = {(c[0], c[1]) for c in table}
    assert (1, 1) in shapes and (2, 2) in shapes
    assert any(h == 1 and w > 1 for h, w in shapes) and any(w == 1 and h > 1 for h, w in shapes)
    assert any(c[5] > helpers.MAX_FUSED for c in table)
    assert {"constant", "binary", "repeat"} <= {c[3] for c in table}
    imgs = exact_images("repeat", 37, 45, 4)
    assert all(np.array_equal(imgs[0], imgs[b]) for b in range(4))
    assert np.unique(exact_images("binary", 45, 52, 1)).tolist() == [0, 255]


def test_renumbering_key_bound():
    src = open(os.path.join(ROOT, "dsrg_b200", "csrc", "common.cuh")).read()
    assert int(re.search(r"constexpr int kNoKey = (0x[0-9A-Fa-f]+);", src).group(1), 16) == K_NO_KEY
    assert renum_key_limit(RENUM_MAX_H_W1, 1) < K_NO_KEY <= renum_key_limit(RENUM_MAX_H_W1 + 1, 1)
    assert RENUM_MAX_H_W1 + 1 == 11140945
    assert RENUM_MAX_H_W1 * 1 <= 1 << 24                 # the pixel-count check alone would let these through
    for W in (2, 3, 32, 33, 4096):                        # wider images with the most pixels stay below it
        assert renum_key_limit((1 << 24) // W, W) < K_NO_KEY


def test_engine_creation_refuses_overflowing_renumbering_keys():
    """The shape check comes before any CUDA call, so it holds without a GPU."""
    L = _lib.lib()
    for H, W in ((RENUM_MAX_H_W1 + 1, 1), ((1 << 24) - 1, 1), (1 << 24, 1)):
        assert not L.dsrg_engine_create(0, 1, H, W, 21)
        assert "bad engine shape" in L.dsrg_last_error().decode(), (H, W)
    if L.dsrg_device_count() > 0:
        return                                            # would allocate a real engine of 11 M pixels
    assert not L.dsrg_engine_create(0, 1, RENUM_MAX_H_W1, 1, 21)
    assert "bad engine shape" not in L.dsrg_last_error().decode()
