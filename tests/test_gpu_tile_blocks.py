"""The per-tile weight and local-index blocks (tiles.cu: tl_w, tl_li), which the forward mean-field kernels bulk-copy
into their shared tables, against the planar weights wn and local indices tl_loc of the same build
(test_gpu_lattice_exact.py checks those against the oracle): slot t of row r of a tile's block is the tile's pixel t,
and a slot outside the image holds weight 0 and 0xFFFF.  Smooth, photo-like and noise images (tiles on the
shared-memory, hybrid and direct paths), both lattices, a second batch on the same engine (the shared spatial
lattice is not rebuilt) and a smaller image size; the width 321 makes 30-pixel tiles and a one-row last tile row."""
import ctypes as C

import numpy as np
import pytest

import helpers
from helpers import tile_geometry, tile_of_pixels
from dsrg_b200 import _lib, api

pytestmark = pytest.mark.gpu
REMOTE = 0xFFFF    # common.cuh: kLocRemote


def planar(eng, which, b):
    """dsrg_engine_tile_views: loc [d+1][N] and wn [d+1][N]."""
    dp1, N = 3 if which == 0 else 6, eng.H * eng.W
    loc, wn = np.zeros((dp1, N), np.uint16), np.zeros((dp1, N), np.float32)
    _lib.check(_lib.lib().dsrg_engine_tile_views(C.c_void_p(eng.h), which, b, None, None, None,
                                                 C.c_void_p(loc.ctypes.data), C.c_void_p(wn.ctypes.data)))
    return loc, wn


def blocks(eng, which, b):
    """dsrg_engine_tile_blocks: w and loc [ntiles][d+1][256]."""
    tiles_x, _, tiles_y = tile_geometry(eng.H, eng.W)
    shape = (tiles_x * tiles_y, 3 if which == 0 else 6, 256)
    w, loc = np.full(shape, np.nan, np.float32), np.zeros(shape, np.uint16)
    _lib.check(_lib.lib().dsrg_engine_tile_blocks(C.c_void_p(eng.h), which, b, C.c_void_p(w.ctypes.data),
                                                  C.c_void_p(loc.ctypes.data)))
    return w, loc


def check_blocks(eng, which, b):
    loc_p, wn_p = planar(eng, which, b)
    w, loc = blocks(eng, which, b)
    tile_of, slot = tile_of_pixels(eng.H, eng.W)
    want_w, want_loc = np.zeros_like(w), np.full_like(loc, REMOTE)
    want_w[tile_of, :, slot] = wn_p.T
    want_loc[tile_of, :, slot] = loc_p.T
    assert np.array_equal(w.view(np.uint32), want_w.view(np.uint32)), ("weights", which, b)
    assert np.array_equal(loc, want_loc), ("local indices", which, b)
    return int((loc_p != REMOTE).sum())


def run_pass(torch, eng, images):
    B, H, W = images.shape[:3]
    un = torch.zeros((B, H, W, eng.M), device="cuda")
    eng.crf_dev(un, torch.from_numpy(images).cuda(), api.crf_params(1.0, maxiter=1), torch.empty_like(un))
    torch.cuda.synchronize()


@pytest.mark.parametrize("kind", ["smooth", "photo", "noise"])
def test_blocks_match_the_planar_views(torch_cuda, kind):
    torch = torch_cuda
    B, H, W = 8, 321, 321
    eng = api.Engine(B, H, W, 21)
    for k, (h, w) in enumerate([(H, W), (H, W), (97, 130)]):
        eng.set_size(h, w)
        run_pass(torch, eng, helpers.seeded_images(h, w, [kind] * B, 300 + 10 * k))
        local = check_blocks(eng, 0, 0)
        assert local > 0
        for b in range(B):
            check_blocks(eng, 1, b)
    eng.close()


def test_blocks_read_out_refusals(torch_cuda):
    eng = api.Engine(2, 41, 41, 21)
    L = _lib.lib()
    for which, b in ((2, 0), (-1, 0), (1, 2), (1, -1)):
        assert L.dsrg_engine_tile_blocks(C.c_void_p(eng.h), which, b, None, None) == _lib.E_INVALID
    eng.close()
    eng = api.Engine(1, 41, 41, 81)   # the label-chunked path builds no tile views
    assert L.dsrg_engine_tile_blocks(C.c_void_p(eng.h), 1, 0, None, None) == _lib.E_STATE
    eng.close()
