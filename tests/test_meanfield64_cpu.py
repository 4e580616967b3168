"""The float64 mean field (oracle/meanfield64.py) and the per-iteration bar of test_gpu_meanfield64.py (no GPU needed).

* The restatement is the oracle: in float32 with the sequential splat its filter equals OracleLattice.compute bit for
  bit, and its marginals equal oracle_crf_inference to a few ulp (numpy's exp is not glibc's expf).
* The bar of a case after n iterations is helpers.BAR_K times the largest float32 model error, at least
  helpers.BAR_FLOOR (the reasoning is in helpers.py).  Every case's bar is printed against the suite's old 1e-4.
* The bar is sensitive: small errors a rewrite of the mean-field kernels could make, applied to the float32
  restatement (meanfield64.MUTANTS), exceed it.  Two of them do not: one more rounding of a slice weight and an
  uncorrected exp2 are each one rounding of the size of the float32 noise itself, so no bar derived from that noise
  can see them; they are printed, not claimed.
* The case table of the GPU test reaches every mean-field path (tile kinds predicted from the oracle's lattices for
  an H100 SXM's 132 SMs, blur branches from meanfield.cu's threshold).
"""
import numpy as np
import pytest

import helpers
from helpers import (BAR_FLOOR, FUSED_CONFIGS, MF64_ITERS, MF64_PATH_CONFIG, MF64_TINY, MF64_TINY_M, MF64_TINY_SEED,
                     MF64_WIDE_M, MF64_ZERO_W, MF64_ZERO_W_M, MAX_FUSED, fused_images, log_unary,
                     mf64_problem_params, mf64_truth_and_bar, oracle_batch, small_image, wide_images)
from oracle import meanfield64

SMS = 132
OLD_TOL = 1e-4
ULP = 2.0 ** -24            # the spacing of float32 values in [0.5, 1)
RESTATEMENT_ULPS = 8        # numpy's rounded float64 exp against glibc's expf, over 10 iterations
CLAIMED = ("axes_reversed", "phantom_missing", "values_fp16")
NOT_CLAIMED = ("weight_rounded", "exp2_uncorrected")


def tiny_image(H, W, img):
    return small_image(np.random.RandomState(MF64_TINY_SEED), H, W, img)


def cpu_cases():
    """(name, image, sf, M, zeroed weight, unary seed) of the CPU table: every fused configuration at a few M,
    the wide path, the tiny shapes and the single-lattice cases of the small paths."""
    out = []
    for img, sf in FUSED_CONFIGS:
        im = fused_images(img)[0]
        for M in (1, 2, 6, 21, 32):
            out.append(("%s sf%g" % (img, sf), im, sf, M, None, 10 * M))
    for img in ("smooth", "noise"):
        for M in MF64_WIDE_M:
            out.append(("wide %s" % img, wide_images(img)[0], 1.0, M, None, M))
    for H, W, img in MF64_TINY:
        out.append(("tiny %dx%d" % (H, W), tiny_image(H, W, img), 1.0, MF64_TINY_M, None, 3))
    for path, zero in MF64_ZERO_W:
        if path in MF64_PATH_CONFIG:
            img, sf = MF64_PATH_CONFIG[path]
            out.append(("%s %s=0" % (path, zero), fused_images(img)[0], sf, MF64_ZERO_W_M[path], zero, 77))
    return out


@pytest.fixture(scope="module")
def table():
    """Per case: the float64 marginals, the bar, the model spread and the float32 runs of every mutant."""
    rows = []
    problems = {}
    for name, im, sf, M, zero, seed in cpu_cases():
        key = (name.split(" M")[0], sf, zero, im.shape)
        if key not in problems:
            problems[key] = meanfield64.Problem(im, mf64_problem_params(sf, zero))
        P = problems[key]
        un = log_unary(1, im.shape[0], im.shape[1], M, seed=seed)[0]
        q64, bar, spread, muts = mf64_truth_and_bar(P, un, extra=[dict(mutant=m) for m in meanfield64.MUTANTS])
        err = {m: {n: float(np.abs(q[n] - q64[n]).max()) for n in MF64_ITERS} for m, q in zip(meanfield64.MUTANTS, muts)}
        rows.append((name, M, bar, spread, err))
    return rows


@pytest.mark.parametrize("img,sf", FUSED_CONFIGS + [("tiny", 1.0)])
def test_restatement_filter_is_the_oracles(img, sf):
    """Splat, blur and slice in float32 with the sequential splat equal OracleLattice.compute bit for bit, in the seq
    form (value size 1, 2) and the SSE form (3 and more), on both lattices."""
    ims = [tiny_image(H, W, k) for H, W, k in MF64_TINY] if img == "tiny" else [fused_images(img)[0]]
    for im in ims:
        P = meanfield64.Problem(im, mf64_problem_params(sf))
        for vs in (1, 2, 3, 7, 24):
            x = np.random.RandomState(vs).rand(P.N, vs).astype(np.float32)
            for k, L in enumerate(P.lattices):
                want = P.crf.lattice(k).compute(x, "sse" if vs > 2 else "seq")
                assert np.array_equal(L.filter(x, np.float32), want), (img, im.shape, vs, k)
        n64, n32 = P.norms(np.float64), P.norms(np.float32)
        for k in range(2):
            assert np.array_equal(n32[k], P.crf.norm(k)), (img, k)
            assert float(np.abs(n64[k] - n32[k]).max() / n64[k].max()) < 2 ** -22


@pytest.mark.parametrize("img,sf", FUSED_CONFIGS)
def test_restatement_inference_is_the_oracles(img, sf):
    """Q after n iterations within RESTATEMENT_ULPS float32 ulps of [0.5, 1) of oracle_crf_inference: the signs,
    norms, alpha, axis order and Potts compatibility are the oracle's; only exp is rounded differently."""
    im = fused_images(img)[:1]
    P = meanfield64.Problem(im[0], mf64_problem_params(sf))
    worst = 0.0
    for M in (1, 2, 3, 21, 35):
        un = log_unary(1, im.shape[1], im.shape[2], M, seed=M)
        q32 = P.run(un[0], 10, np.float32)
        for n in (0, 1, 2, 3, 10):
            d = float(np.abs(q32[n] - oracle_batch(im, un, sf, n)[0]).max()) / ULP
            worst = max(worst, d)
            assert d <= RESTATEMENT_ULPS, (img, sf, M, n, d)
    print("\n%s sf%g: restatement vs oracle_crf_inference, worst %.1f ulp" % (img, sf, worst))


def test_every_bar_is_far_under_the_old_tolerance(table):
    print("\n%-18s %4s  " % ("case", "M") + "  ".join("n=%-2d bar  (1e-4/bar)" % n for n in MF64_ITERS))
    for name, M, bar, spread, _ in table:
        print("%-18s %4d  " % (name, M) + "  ".join("%.2e (%5.0fx)" % (bar[n], OLD_TOL / bar[n]) for n in MF64_ITERS))
        assert all(bar[n] >= BAR_FLOOR for n in MF64_ITERS)
        for n in (1, 2, 3):
            assert bar[n] <= OLD_TOL / 4, (name, M, n, bar[n])
        assert bar[10] <= OLD_TOL, (name, M, bar[10])


def test_mutants_exceed_the_bar(table):
    """Each claimed mutant exceeds the bar on at least one case; the table shows by how much, and which mutants the
    old bar (1e-4 after ten iterations) lets through everywhere."""
    assert set(CLAIMED) | set(NOT_CLAIMED) == set(meanfield64.MUTANTS)
    print("\n%-18s  worst err/bar over the table (case, M, n)   caught by 1e-4 at n=10" % "mutant")
    for m in meanfield64.MUTANTS:
        ratio, where = max(((err[m][n] / bar[n], (name, M, n)) for name, M, bar, _, err in table for n in MF64_ITERS),
                           key=lambda r: r[0])
        old = any(err[m][10] > OLD_TOL for _, _, _, _, err in table)
        print("%-18s  %10.1f  %-28s  %s%s" % (m, ratio, where, "yes" if old else "NO, passes",
                                             "" if m in CLAIMED else "   (not claimed)"))
        if m in CLAIMED:
            assert ratio > 1.0, (m, ratio, where)
        else:
            assert ratio <= 1.0, ("%s is caught now: move it to CLAIMED" % m, ratio, where)


def test_device_model_sits_under_the_bar(table):
    """The model of the device's arithmetic is one of the five the bar is taken over, so the device's own rounding
    differences alone can never exceed it; here the four oracle-arithmetic models alone give the bar, and the device
    model stays within it."""
    # recomputed on one case per path: the spread of the oracle models alone against the device model's error
    for img, sf in FUSED_CONFIGS:
        im = fused_images(img)[0]
        P = meanfield64.Problem(im, mf64_problem_params(sf))
        un = log_unary(1, im.shape[0], im.shape[1], 21, seed=5)[0]
        q64, _, _, runs = mf64_truth_and_bar(P, un, extra=[dict(splat_order=s) for s in (None, 1, 2, 3)] +
                                             [dict(splat_order=9, arith="device")])
        for n in MF64_ITERS:
            oracle_spread = max(float(np.abs(r[n] - q64[n]).max()) for r in runs[:4])
            dev = float(np.abs(runs[4][n] - q64[n]).max())
            assert dev <= max(helpers.BAR_K * oracle_spread, BAR_FLOOR), (img, sf, n, dev, oracle_spread)


# ---- the GPU test's case table reaches every path ----
def test_fused_cases_reach_every_tile_path():
    kinds = {}
    for img, sf in FUSED_CONFIGS:
        p = helpers.predict_tile_paths(fused_images(img), sf, SMS)
        kinds[(img, sf)] = (set(p["sp"]), set(p["bi"].ravel()))
    assert kinds[MF64_PATH_CONFIG["smem"]] == ({"smem"}, {"smem"})
    assert "direct" in kinds[MF64_PATH_CONFIG["bi_direct"]][1]
    assert "direct" in kinds[MF64_PATH_CONFIG["sp_direct"]][0]
    assert {helpers.padded(M) for M in helpers.FUSED_ITER_M} == set(range(4, MAX_FUSED + 1, 4))
    assert {helpers.tail1(M) for M in helpers.FUSED_ITER_M} == {True, False}


def test_hybrid_gate_and_switch_cases_reach_their_paths():
    image = helpers.hybrid_images()
    assert helpers.predict_tile_paths(image, 1.0, SMS)["hybrid_tiles"] > 0
    g2 = helpers.seeded_images(*helpers.GATE2_SHAPE, ("noise", "noise"), helpers.GATE2_SEED)
    assert helpers.blur_branch(*helpers.GATE2_SHAPE, [helpers.bilateral_vertices(im) for im in g2]) == "gate2"
    assert set(MF64_ZERO_W_M) == {"smem", "bi_direct", "sp_direct", "hybrid", "wide"}
    assert {c[-1] for c in helpers.SWITCH_CASES} == {"ungated", "gate1", "gate2"}
    assert set(helpers.MF64_GATE2_M) <= set(helpers.GATE2_M)
    assert {helpers.padded(M) for M in helpers.MF64_GATE2_M} >= {8, 24, 32}


def test_wide_and_tiny_cases():
    assert MF64_WIDE_M == [33, 128, 255] and all(M > MAX_FUSED for M in MF64_WIDE_M)
    assert MF64_ZERO_W_M["wide"] > MAX_FUSED
    assert sorted((H * W) % 4 for H, W, _ in MF64_TINY) == [0, 1, 2, 3]
    for H, W, img in MF64_TINY:                    # tiny images are one tile and one ungated blur
        assert helpers.blur_branch(H, W, [helpers.bilateral_vertices(tiny_image(H, W, img))]) == "ungated"
    # the 41 x 41 noise image (N % 4 = 1) has vertices only the phantom lanes touch, and they carry mass
    P = meanfield64.Problem(fused_images("noise")[0], mf64_problem_params(1.0))
    L = P.lattices[1]
    real = np.zeros(L.V + 1, bool)
    real[L.rows] = True
    assert (~real[1:]).sum() > 0
