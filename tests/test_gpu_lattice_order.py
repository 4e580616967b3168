"""GPU tests of the lattice's vertex numbering (csrc/lattice.cu): the ids are a permutation of 0..V-1 ordered by
each vertex's first incidence in tile-major pixel order, the blur neighbours are the oracle's under that mapping, and
two builds of the same images give the same tables."""
import numpy as np
import pytest

from helpers import csrc_constants, tile_geometry
from dsrg_b200 import api, synth
from oracle import crf_oracle

pytestmark = pytest.mark.gpu

CASES = ((41, 41, 12.0, "smooth"), (37, 53, 1.0, "noise"), (64, 64, 1.0, "smooth"), (50, 70, 12.0, "photo"))


def tile_major_pos(H, W):
    """Position of every pixel (row-major order) in tile-major order: tile index, then thread index in the tile."""
    k = csrc_constants()
    tiles_x, tile_w, _ = tile_geometry(H, W)
    ys, xs = np.mgrid[0:H, 0:W]
    tx, ty = xs // tile_w, ys // k["kTileH"]
    tid = (ys - ty * k["kTileH"]) * k["kTileW"] + (xs - tx * tile_w)
    return ((ty * tiles_x + tx) * k["kTileW"] * k["kTileH"] + tid).ravel()


def run_crf(eng, batch, sf):
    import torch
    unary = torch.from_numpy(np.transpose(batch["probs"], (0, 2, 3, 1)).copy()).cuda()
    eng.crf_dev(unary, torch.from_numpy(batch["image"]).cuda(), api.crf_params(sf, maxiter=1), torch.empty_like(unary))


def check_order(off, H, W):
    """ids follow the first tile-major incidence; vertices without one (the phantom lanes') come last.
    Returns the number of vertices that pixels touch."""
    dp1 = off.shape[0]
    ids = off - 1
    key = tile_major_pos(H, W)[None, :] * dp1 + np.arange(dp1)[:, None]
    V_pix = int(ids.max()) + 1
    first = np.full(V_pix, np.iinfo(np.int64).max)
    np.minimum.at(first, ids.ravel(), key.ravel())
    assert (first < np.iinfo(np.int64).max).all(), "ids touched by pixels are not contiguous from 0"
    assert (np.diff(first) > 0).all(), "ids do not increase with the first tile-major incidence"
    return V_pix


def check_against_oracle(off, nbr, lat, V_pix):
    """The engine's tables are the oracle's lattice renamed: one-to-one vertex mapping, same neighbours."""
    dp1, V = off.shape[0], nbr.shape[1] - 1
    assert V == lat.M
    o = lat.offset.T                                   # (d+1, N) oracle ids
    m = np.full(lat.M, -1, np.int64)
    m[o.ravel()] = off.ravel() - 1
    assert np.array_equal(m[o], off - 1), "a vertex maps to two ids"
    seen = m >= 0
    assert np.unique(m[seen]).size == seen.sum() == V_pix
    assert (nbr[:, 0] == 0).all(), "the zero row must point at itself"
    for j in range(dp1):
        for on, col in ((lat.n1[j], 0), (lat.n2[j], 1)):
            got = nbr[j, m[seen] + 1, col]
            tgt = on[seen]
            want = np.where(tgt < 0, 0, m[np.maximum(tgt, 0)] + 1)
            mapped = (tgt < 0) | (m[np.maximum(tgt, 0)] >= 0)
            assert np.array_equal(got[mapped], want[mapped]), "axis %d neighbour %d" % (j, col)
            # a neighbour that no pixel touches is one of the phantom lanes' vertices, numbered last
            assert (got[~mapped] > V_pix).all()


@pytest.mark.parametrize("H,W,sf,img", CASES)
def test_numbering_is_tile_major_and_matches_the_oracle(torch_cuda, H, W, sf, img):
    B, M = 2, 21
    batch = synth.make_batch(B, H, W, image=img, start=5)
    eng = api.Engine(B, H, W, M)
    run_crf(eng, batch, sf)
    vs, vb = eng.lattice_sizes(B)
    for b in range(B):
        c = crf_oracle.DenseCRF(W, H, M)
        c.set_unary_energy(np.zeros(H * W * M, np.float32))
        c.add_pairwise_energy(10, 80 / sf, 80 / sf, 13, 13, 13, 3, 3 / sf, 3 / sf, batch["image"][b].ravel())
        for which in (0, 1):
            if which == 0 and b > 0:
                continue                               # one spatial lattice serves the batch
            off, nbr = eng.lattice_tables(which, b)
            assert nbr.shape[1] - 1 == (vs if which == 0 else vb[b])
            V_pix = check_order(off, H, W)
            check_against_oracle(off, nbr, c.lattice(which), V_pix)
    eng.close()


def test_two_builds_give_identical_tables(torch_cuda):
    B, H, W, sf = 3, 57, 66, 1.0
    batch = synth.make_batch(B, H, W, image="photo", start=9)
    tables = []
    for _ in range(2):
        eng = api.Engine(B, H, W, 21)
        for _ in range(2):                             # the second call rebuilds the bilateral lattice in place
            run_crf(eng, batch, sf)
            tables.append([eng.lattice_tables(w, b) for w in (0, 1) for b in range(B)])
        eng.close()
    for t in tables[1:]:
        for (o0, n0), (o1, n1) in zip(tables[0], t):
            assert np.array_equal(o0, o1) and np.array_equal(n0, n1)
