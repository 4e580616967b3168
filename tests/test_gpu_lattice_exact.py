"""The lattice build (csrc/lattice.cu, tiles.cu), table by table, against the oracle (crf_oracle.DenseCRF(...).lattice,
pinned to the reference's permutohedral.cpp by test_oracle_golden.py, and the reference's own lattice where
oracle/_ref was built): per image and per lattice the vertex count, the offsets and blur neighbours under the
one-to-one vertex mapping, the barycentric weights bit for bit, the norms against the float64 norms, the weights
wn = bary * norm, and the tile-local views restated in numpy.  After every pass the build must leave the state the
next one starts from: every hash slot empty, hval -1 and vkey kNoKey, over the whole allocation.

Cases: bench.py's batch (64 distinct 321 x 321 images) at both scale factors and three kinds of image, 513 x 513, a
COCO-sized image on the label-chunked path, strips and tiny shapes with 0..3 phantom lanes, a constant image, a
0/255 image, a repeated image, the sigmas at the edge of the packed-key range and one float32 step past it, and a
sequence of builds on one engine (other images, a smaller batch, set_size down and up, a new scale factor, graph
replays over new image contents).  The module prints each case's vertex counts, V/capv, largest |key| and wall time.
"""
import ctypes as C
import os
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import helpers
from helpers import (EDGE_B, EDGE_BI, EDGE_MAX_KEY, EDGE_SHAPE, EDGE_SP, EXACT_BENCH, EXACT_BENCH_CONFIGS,
                     EXACT_BENCH_FULL, EXACT_CASES, check_against_oracle, check_order, csrc_constants,
                     demote_hybrid_tiles, edge_params, exact_images, hybrid_tiles_on, lattice_features,
                     lattice_sigmas, lattice_tile_kinds, max_abs_key, phantom_lanes, tile_geometry, tile_of_pixels)
from dsrg_b200 import _lib, api
from oracle import crf_oracle, meanfield64

pytestmark = pytest.mark.gpu
ROWS = []          # (case, lattice, V min, V max, max V/capv, max |key|, seconds)
REMOTE = 0xFFFF    # common.cuh: kLocRemote
HYBRID = 1 << 16   # common.cuh: kTileHybrid


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    if not ROWS:
        return
    print("\n%-26s %-9s %9s %9s %8s %8s %8s" % ("case", "lattice", "V min", "V max", "V/capv", "max|key|", "seconds"))
    for case, which, vmin, vmax, ratio, key, sec in ROWS:
        print("%-26s %-9s %9d %9d %8.4f %8d %8.1f" % (case, ("spatial", "bilateral")[which], vmin, vmax, ratio, key,
                                                       sec))


def sm_count(torch):
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def run_pass(torch, eng, images, params, host=False):
    """One mean-field iteration over `images`: what matters here is the lattices it builds."""
    B, H, W = images.shape[:3]
    if host:   # the host entry point also reads the device's key-range flag back
        eng.crf_host(np.zeros((B, H, W, eng.M), np.float32), images, params)
        return
    un = torch.zeros((B, H, W, eng.M), device="cuda")
    eng.crf_dev(un, torch.from_numpy(images).cuda(), params, torch.empty_like(un))
    torch.cuda.synchronize()


def tile_views(eng, which, b, views=True):
    """dsrg_engine_tile_views: (nloc, hy, hdr, loc, wn), or only wn."""
    k = csrc_constants()
    tiles_x, _, tiles_y = tile_geometry(eng.H, eng.W)
    nt, dp1, N = tiles_x * tiles_y, 3 if which == 0 else 6, eng.H * eng.W
    maxloc = k["DSRG_MAXLOC_SP"] if which == 0 else k["DSRG_MAXLOC_HY"]
    out = [np.zeros(nt, np.int32), np.zeros(nt, np.uint8), np.zeros((nt, maxloc, 2), np.int32),
           np.zeros((dp1, N), np.uint16), np.zeros((dp1, N), np.float32)]
    ptrs = [C.c_void_p(a.ctypes.data) if views or i == 4 else None for i, a in enumerate(out)]
    _lib.check(_lib.lib().dsrg_engine_tile_views(C.c_void_p(eng.h), which, b, *ptrs))
    return out if views else out[4]


def check_tiles(views, off, H, W, kinds, built):
    """The tile-local views restated: which tiles have a list (and which of those are hybrid) is `kinds`
    (helpers.lattice_tile_kinds after k_tile_demote), `built` the kinds k_tile_build gave them; a plain tile lists
    exactly the distinct rows of its pixels, a hybrid one the most-touched of them; every local (r, pixel) points at
    the entry of its row; segment lengths are the incidence counts, do not increase, and start where the
    even-rounded lengths before them end."""
    nloc, hy, hdr, loc, _ = views
    nt, maxloc = hdr.shape[:2]
    tile_of, _ = tile_of_pixels(H, W)
    listed = nloc >= 0
    hybrid = listed & ((nloc & HYBRID) != 0)
    plain = listed & ~hybrid
    cnt = np.where(listed, nloc & 0xFFFF, 0)
    assert np.array_equal(np.where(hybrid, "hybrid", np.where(listed, "smem", "direct")).astype(object), kinds)
    assert np.array_equal(hy, hybrid.astype(np.uint8))
    assert (cnt <= maxloc).all()
    t = np.broadcast_to(tile_of, off.shape)
    local = loc != REMOTE
    # k_mf_tile's direct path reads off, not tl_loc: an overflow tile built without a list marks every incidence
    # remote, one that k_tile_demote took off the hybrid list keeps its hybrid view
    assert not local[(built == "direct")[t]].any(), "an overflow tile without a list has a local incidence"
    assert local[plain[t]].all(), "a plain tile has a remote incidence"
    local &= listed[t]
    li, lt = loc[local].astype(np.int64), t[local]
    assert (li < cnt[lt]).all()
    assert np.array_equal(hdr[lt, li, 1], off[local]), "a local incidence points at another row"
    inc = np.zeros((nt, maxloc), np.int64)
    np.add.at(inc, (lt, li), 1)
    seg, first = hdr[:, :, 0] >> 16, hdr[:, :, 0] & 0xFFFF
    valid = np.arange(maxloc)[None, :] < cnt[:, None]
    assert np.array_equal(seg[valid], inc[valid]) and (seg[valid] > 0).all()
    assert (np.diff(seg, axis=1)[valid[:, 1:]] <= 0).all(), "segment lengths increase"
    even = np.where(valid, (seg + 1) & ~1, 0)
    assert np.array_equal(first[valid], (np.cumsum(even, 1) - even)[valid])
    R = int(off.max()) + 1
    u, ucnt = np.unique(t.astype(np.int64) * R + off, return_counts=True)
    utile = u // R
    assert np.array_equal(np.bincount(utile, minlength=nt)[plain], cnt[plain]), "a plain tile misses a row"
    if hybrid.any():   # a hybrid tile keeps its most-touched vertices
        kept = np.isin(u, (np.arange(nt)[:, None] * R + hdr[:, :, 1])[valid & hybrid[:, None]])
        lo = np.full(nt, np.iinfo(np.int64).max)
        hi = np.zeros(nt, np.int64)
        np.minimum.at(lo, utile[kept], ucnt[kept])
        np.maximum.at(hi, utile[~kept], ucnt[~kept])
        assert (lo[hybrid] >= hi[hybrid]).all()


def image_problem(image, params):
    """The oracle's lattices of one image (meanfield64.Problem keeps them and gives the float64 norms)."""
    return meanfield64.Problem(image, params)


def norm_bar(P, which):
    n64 = P.norms(np.float64)[which]
    spread = max(float(np.abs(P.norms(np.float32, s)[which] - n64).max() / n64.max()) for s in (None, 1, 2, 3))
    return n64, max(helpers.BAR_K * spread, 2.0 ** -23)


def check_image(eng, b, image, params, P, which, norm):
    """Image b's lattice `which` against the oracle, table by table.  Returns its engine tables (for comparisons
    between images) and its largest |key|."""
    H, W = image.shape[:2]
    lat = P.crf.lattice(which)
    off, nbr = eng.lattice_tables(which, b)
    V_pix = check_order(off, H, W)
    check_against_oracle(off, nbr, lat, V_pix)
    bary = eng.lattice_bary(which, b)
    assert np.array_equal(bary.view(np.uint32), np.ascontiguousarray(lat.bary.T).view(np.uint32)), \
        "barycentric weights differ from the oracle's (%d of %d)" % ((bary != lat.bary.T).sum(), bary.size)
    sigma = lattice_sigmas(params, which)
    if crf_oracle.ref_available():
        ref = crf_oracle.RefLattice(lattice_features(image, sigma)[:H * W])
        check_against_oracle(off, nbr, ref, V_pix)
        assert np.array_equal(bary.view(np.uint32), np.ascontiguousarray(ref.bary.T).view(np.uint32))
    n64, bar = norm_bar(P, which)
    rel = float(np.abs(norm - n64).max() / n64.max())
    assert rel <= bar, (which, b, rel, bar)
    wn = tile_views(eng, which, b, views=False)
    assert np.array_equal(wn.view(np.uint32), (bary * norm[None, :]).view(np.uint32)), "wn is not bary * norm"
    return (off, nbr, bary, norm, wn), max_abs_key(image, sigma)


def check_pass(torch, eng, name, images, params, full, t0):
    """Everything the last pass over `images` built: V of every image, the full tables of the images in `full`,
    the tile-local views and the hybrid-tile count, and the idle state of both lattice families."""
    B, H, W = images.shape[:3]
    N, P_ = H * W, phantom_lanes(H * W)
    fused = eng.M <= helpers.MAX_FUSED
    sms = sm_count(torch)
    gate = fused and hybrid_tiles_on(H, W, B, sms)
    full = sorted(set(full))

    def oracle(b):
        P = image_problem(images[b], params)
        if b in full:
            for which in (0, 1):   # the norms' float64 and float32 runs, while the thread holds no GIL-bound work
                norm_bar(P, which)
        kinds = lattice_tile_kinds(P.crf.lattice(1).offset, H, W, 1, gate) if fused else None
        sp = P.crf.lattice(0).M if b == 0 else None
        sp_kinds = lattice_tile_kinds(P.crf.lattice(0).offset, H, W, 0, False) if fused and b == 0 else None
        return P.crf.lattice(1).M, kinds, sp, sp_kinds, (P if b in full else None)

    with ThreadPoolExecutor(min(B, os.cpu_count() or 1, 16)) as ex:
        res = list(ex.map(oracle, range(B)))
    vs, vb = eng.lattice_sizes(B)
    assert vs == res[0][2]
    assert np.array_equal(vb, [r[0] for r in res]), "bilateral vertex counts differ from the oracle's"
    ns, nb = eng.norms(B)
    tables, keys = {}, {0: 0, 1: 0}
    if fused:
        bi_built = np.stack([r[1] for r in res])
        bi_kinds = bi_built.copy()
        nhy = demote_hybrid_tiles(bi_kinds, sms)
        assert eng.hybrid_tiles == nhy
    else:
        with pytest.raises(_lib.DsrgError) as ei:
            tile_views(eng, 1, 0)
        assert ei.value.code == _lib.E_STATE
    for b in full:
        P = res[b][4]
        for which in (0, 1) if b == full[0] else (1,):   # one spatial lattice serves the batch
            t, key = check_image(eng, b, images[b], params, P, which, ns if which == 0 else nb[b])
            tables[(which, b)] = t
            keys[which] = max(keys[which], key)
            if fused:
                kinds = (res[0][3], res[0][3]) if which == 0 else (bi_kinds[b], bi_built[b])
                check_tiles(tile_views(eng, which, b), t[0], H, W, *kinds)
    for which in (0, 1):
        assert eng.lattice_idle(which) == (0, 0, 0), (name, which, eng.lattice_idle(which))
    sec = time.time() - t0
    ROWS.append((name, 0, vs, vs, vs / ((N + P_) * 3.0), keys[0], sec))
    ROWS.append((name, 1, int(vb.min()), int(vb.max()), float(vb.max()) / ((N + P_) * 6.0), keys[1], sec))
    return tables, keys


@pytest.mark.parametrize("img,sf", EXACT_BENCH_CONFIGS)
def test_bench_batch(torch_cuda, img, sf):
    H, W, B = EXACT_BENCH
    t0 = time.time()
    images = helpers.seeded_images(H, W, [img] * B, 900)
    eng = api.Engine(B, H, W, 21)
    params = api.crf_params(sf, maxiter=1)
    run_pass(torch_cuda, eng, images, params)
    check_pass(torch_cuda, eng, "bench %s sf %g" % (img, sf), images, params, EXACT_BENCH_FULL, t0)
    eng.close()


@pytest.mark.parametrize("name", list(EXACT_CASES))
def test_case(torch_cuda, name):
    H, W, B, kind, sf, M, _, _ = EXACT_CASES[name]
    t0 = time.time()
    images = exact_images(kind, H, W, B)
    eng = api.Engine(B, H, W, M)
    params = api.crf_params(sf, maxiter=1)
    run_pass(torch_cuda, eng, images, params)
    tables, _ = check_pass(torch_cuda, eng, name, images, params, range(B), t0)
    if kind == "repeat":
        # one image B times: the same offsets, neighbours and weights (the norms add in atomic order, and a tile
        # numbers its vertices of equal segment length in arrival order), the same tiles listing the same rows
        def listed_rows(b):
            nloc, hy, hdr, _, _ = tile_views(eng, 1, b)
            cnt = np.where(nloc >= 0, nloc & 0xFFFF, 0)
            t, l = np.nonzero(np.arange(hdr.shape[1])[None, :] < cnt[:, None])
            e = np.stack([t, hdr[t, l, 1], hdr[t, l, 0] >> 16])
            return nloc, hy, e[:, np.lexsort(e[::-1])]

        for b in range(1, B):
            for a0, a1 in zip(tables[(1, 0)][:3], tables[(1, b)][:3]):
                assert np.array_equal(a0, a1), b
            for a0, a1 in zip(listed_rows(0), listed_rows(b)):
                assert np.array_equal(a0, a1), b
    eng.close()


def test_key_range_edge(torch_cuda):
    """At the sigmas where key_range_ok only just passes the tables still match and the device's flag stays clear
    (crf_host reads it back); one float32 step below is refused before any launch, and the engine goes on."""
    torch = torch_cuda
    H, W = EDGE_SHAPE
    t0 = time.time()
    images = exact_images("binary", H, W, EDGE_B)
    eng = api.Engine(EDGE_B, H, W, 21)
    params = edge_params()
    run_pass(torch, eng, images, params, host=True)
    _, keys = check_pass(torch, eng, "key-range edge", images, params, range(EDGE_B), t0)
    assert keys == EDGE_MAX_KEY and keys[1] > 1024
    down = lambda s: float(np.nextafter(np.float32(s), np.float32(0)))   # noqa: E731
    refused = [(EDGE_SP, (down(EDGE_BI[0]),) + EDGE_BI[1:]),     # the spatial lattice is not rebuilt: no launch
               ((down(EDGE_SP[0]), EDGE_SP[1]), EDGE_BI), ((EDGE_SP[0], down(EDGE_SP[1])), EDGE_BI)]
    for k, (sp, bi) in enumerate(refused):
        eng.take_launch_count()
        with pytest.raises(_lib.DsrgError) as ei:
            run_pass(torch, eng, images, edge_params(sp, bi))
        assert ei.value.code == _lib.E_KEYRANGE, k
        assert eng.take_launch_count() == 0, k
        for which in (0, 1):
            assert eng.lattice_idle(which) == (0, 0, 0)
        t0 = time.time()
        images = exact_images("binary", H, W, EDGE_B, seed=k + 1)
        run_pass(torch, eng, images, params, host=True)
        check_pass(torch, eng, "key-range edge, after %d" % k, images, params, range(EDGE_B), t0)
    eng.close()


def test_engine_refuses_overflowing_renumbering_keys(torch_cuda):
    L = _lib.lib()
    for H in (helpers.RENUM_MAX_H_W1 + 1, 1 << 24):
        assert not L.dsrg_engine_create(0, 1, H, 1, 21)
        assert "bad engine shape" in L.dsrg_last_error().decode()
    assert helpers.renum_key_limit(helpers.RENUM_MAX_H_W1 + 1, 1) >= helpers.K_NO_KEY


def test_build_to_build_on_one_engine(torch_cuda):
    """Each build starts from what the last one left: other images at the full batch and a smaller one, set_size down
    and back up, a new scale factor (the spatial lattice is rebuilt), then graph replays on a side stream over new
    image contents in the same buffers."""
    torch = torch_cuda
    maxB, Hc, Wc = 6, 64, 80
    eng = api.Engine(maxB, Hc, Wc, 21)
    steps = [((Hc, Wc), maxB, "photo", 1.0), ((Hc, Wc), 3, "noise", 1.0), ((41, 57), 4, "smooth", 1.0),
             ((Hc, Wc), 5, "photo", 1.0), ((Hc, Wc), 5, "photo", 12.0)]
    for k, ((H, W), B, kind, sf) in enumerate(steps):
        t0 = time.time()
        eng.set_size(H, W)
        images = exact_images(kind, H, W, B, seed=40 + k)
        params = api.crf_params(sf, maxiter=1)
        run_pass(torch, eng, images, params)
        check_pass(torch, eng, "sequence step %d" % (k + 1), images, params, range(B), t0)
    H, W = Hc, Wc
    B = steps[-1][1]
    eng.set_graphs(True)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        d_im = torch.empty((B, H, W, 3), dtype=torch.uint8, device="cuda")
        un = torch.zeros((B, H, W, eng.M), device="cuda")
        out = torch.empty_like(un)
    replays = eng.graph_replays
    for k in range(4):
        t0 = time.time()
        images = exact_images("photo", H, W, B, seed=60 + k)
        with torch.cuda.stream(s):
            d_im.copy_(torch.from_numpy(images))
            eng.crf_dev(un, d_im, params, out, stream=s.cuda_stream)
        s.synchronize()
        check_pass(torch, eng, "graph pass %d" % (k + 1), images, params, range(B), t0)
    assert eng.graph_replays - replays >= 2
    eng.close()
