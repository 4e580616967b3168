"""The CRF at pairwise parameters other than CRF()'s (helpers.PARAM_SETS): anisotropic spatial and bilateral sigmas,
per-channel colour sigmas, other and negative Potts weights, spatial and bilateral sigmas chosen apart to reach tile
paths the scale factor never pairs, sigmas so large that an axis or a colour collapses, and a strip whose x terms sit
at the packed-key limit.  Each of the nine values goes to its own place in the engine (the lattice features, the
key-range check, the spatial-lattice cache, the graph key, the Potts coefficients), and every image is non-square,
so a value sent to the wrong place shows.

Per set: both lattices against the oracle's (and the reference's where oracle/_ref was built) table by table, the
mean field in both unary layouts after 1, 2, 3 and 10 iterations against the float64 restatement under its per-case
bar, on the fused path the set reaches, on a tiny shape with phantom lanes and (two sets) on the label-chunked path.
Entry points: a DenseCRF object, the reference build's DenseCRF, dsrg_forward_dev, crflayer_forward_dev and
predict_mask_dev.  One engine with graphs on walks a sequence of sets that each change one value, against a fresh
graphs-off engine and the oracle's lattices after every call.  The module prints one row per set and path.
"""
import time

import numpy as np
import pytest

from helpers import (KEY_EDGE_B, KEY_EDGE_BI, KEY_EDGE_MAX_KEY, KEY_EDGE_SHAPE, KEY_EDGE_SP, MF64_ITERS, PARAM_M,
                     PARAM_SETS, PARAM_TINY, PARAM_WIDE_M, PARAM_WIDE_SETS, Truth, blur_branch, check_against_oracle,
                     check_order, crf_both_layouts, edge_params, key_range_ok, lattice_features, lattice_sigmas,
                     log_unary, make_params, max_abs_key, oracle_lattices, pairwise_args, param_set_images,
                     predict_tile_paths, set_images, set_params, tile_pairing)
from dsrg_b200 import _lib, api
from oracle import crf_oracle

pytestmark = pytest.mark.gpu
TOL = 1e-4           # the suite's bound on the CRF's float32 marginals (test_gpu_crf.py)
LAT_ROWS = []        # (set, tile paths, blur branch, V spatial, V bilateral min, max, max|key| spatial, bilateral)
MF_ROWS = []         # (set, path, n_iters, device error, bar)


@pytest.fixture(scope="module", autouse=True)
def report():
    t0 = time.time()
    yield
    if LAT_ROWS:
        print("\n%-30s %-14s %-8s %8s %8s %8s %9s %9s" % ("set", "tiles sp/bi", "blur", "V sp", "V bi min", "V bi max",
                                                         "|key| sp", "|key| bi"))
        for r in LAT_ROWS:
            print("%-30s %-14s %-8s %8d %8d %8d %9d %9d" % r)
    if MF_ROWS:
        print("\n%-40s %-14s %3s  %9s  %9s  %5s" % ("set", "path", "n", "dev err", "bar", "ratio"))
        for case, path, n, err, bar in MF_ROWS:
            print("%-40s %-14s %3d  %9.2e  %9.2e  %5.2f" % (case, path, n, err, bar, err / bar))
    print("module wall time %.1f s" % (time.time() - t0))


def sm_count(torch):
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def check(case, path, got, q64, bar, n, images):
    rows = [(float(np.abs(got[b] - q64[b][n]).max()), bar[b][n]) for b in images]
    err, b_bar = max(rows, key=lambda r: r[0] / r[1])
    MF_ROWS.append((case, path, n, err, b_bar))
    for b, (e, bb) in zip(images, rows):
        assert e <= bb, (case, path, n, b, e, bb)


def run_case(torch, case, path, image, unary, params, truth, eng=None):
    """crf_dev in both layouts at every n_iters against the float64 marginals."""
    B, H, W, M = unary.shape
    own = eng is None
    eng = eng or api.Engine(B, H, W, M)
    q64, bar = truth(unary)
    for n in MF64_ITERS:
        p = api.CrfParams.from_buffer_copy(params)
        p.n_iters = n
        nhwc, nchw = crf_both_layouts(torch, eng, unary, image, p)
        check(case, path, nhwc, q64, bar, n, truth.images)
        check(case + " NCHW", path, nchw, q64, bar, n, truth.images)
    if own:
        eng.close()


def check_lattices(eng, images, params, compare):
    """Both lattices of the engine's last pass against the oracle's (and the reference's, where built) under
    `params`: vertex counts, offsets and neighbours under the vertex mapping, barycentric weights bit for bit; both
    lattice families idle afterwards.  Returns (V spatial, V bilateral per image, largest |key| per lattice)."""
    B, H, W = images.shape[:3]
    vs, vb = eng.lattice_sizes(B)
    keys = {0: 0, 1: 0}
    for b in compare:
        c = oracle_lattices(images[b], params)
        for which in (0, 1) if b == compare[0] else (1,):   # one spatial lattice serves the batch
            lat = c.lattice(which)
            assert (vs if which == 0 else vb[b]) == lat.M, (which, b)
            off, nbr = eng.lattice_tables(which, b)
            V_pix = check_order(off, H, W)
            check_against_oracle(off, nbr, lat, V_pix)
            bary = eng.lattice_bary(which, b)
            assert np.array_equal(bary.view(np.uint32), np.ascontiguousarray(lat.bary.T).view(np.uint32)), \
                "lattice %d of image %d: barycentric weights differ from the oracle's" % (which, b)
            sigma = lattice_sigmas(params, which)
            if crf_oracle.ref_available():
                ref = crf_oracle.RefLattice(lattice_features(images[b], sigma)[:H * W])
                check_against_oracle(off, nbr, ref, V_pix)
                assert np.array_equal(bary.view(np.uint32), np.ascontiguousarray(ref.bary.T).view(np.uint32))
            keys[which] = max(keys[which], max_abs_key(images[b], sigma))
    for which in (0, 1):
        assert eng.lattice_idle(which) == (0, 0, 0), which
    return vs, vb, keys


@pytest.mark.parametrize("name", list(PARAM_SETS))
def test_param_set(torch_cuda, name):
    torch = torch_cuda
    image = param_set_images(name)
    B, H, W = image.shape[:3]
    params = set_params(name)
    pred = predict_tile_paths(image, params, sm_count(torch))
    pairing = tile_pairing(pred)
    want = PARAM_SETS[name][5]
    if want is not None:
        assert pairing == want, "%s no longer reaches the tile paths %s (it reaches %s)" % (name, want, pairing)
    path = "%s/%s" % pairing
    compare = list(range(B)) if B <= 2 else [int(np.argmax((pred["bi"] == "hybrid").sum(1)))]
    truth = Truth(image, params, compare)
    eng = api.Engine(B, H, W, PARAM_M)
    run_case(torch, name, path, image, log_unary(B, H, W, PARAM_M, seed=PARAM_M), params, truth, eng)
    assert eng.hybrid_tiles == pred["hybrid_tiles"]
    vs, vb, keys = check_lattices(eng, image, params, compare)
    LAT_ROWS.append((name, path, blur_branch(H, W, vb), vs, int(vb.min()), int(vb.max()), keys[0], keys[1]))
    eng.close()
    if name in PARAM_WIDE_SETS:
        eng = api.Engine(B, H, W, PARAM_WIDE_M)
        run_case(torch, name + " M%d" % PARAM_WIDE_M, "wide", image,
                 log_unary(B, H, W, PARAM_WIDE_M, seed=PARAM_WIDE_M, scale=4.0), params, truth, eng)
        check_lattices(eng, image, params, compare)
        eng.close()
    # a tiny image of the set's kind: one tile, three phantom lanes
    tiny = set_images(PARAM_SETS[name][2], *PARAM_TINY, 2)
    run_case(torch, name + " %dx%d" % PARAM_TINY, "tiny", tiny, log_unary(2, *PARAM_TINY, 5, seed=3), params,
             Truth(tiny, params, range(2)))


@pytest.mark.parametrize("name", ["aniso_xy", "weights", "weights_neg"])
def test_entry_points(torch_cuda, name):
    """dsrg_forward_dev (crf_out) and crflayer_forward_dev (unary: the in-place clamped probs), a DenseCRF object
    (unary energy -log p) against the float64 bar, its map() against the oracle object's, the reference build's
    DenseCRF, and predict_mask_dev with the set's parameters."""
    torch = torch_cuda
    image = param_set_images(name)
    B, H, W = image.shape[:3]
    M = PARAM_M
    params = set_params(name)
    truth = Truth(image, params, range(B))
    rng = np.random.RandomState(11)
    logits = rng.randn(B, M, H, W) * 2
    probs = np.exp(logits - logits.max(1, keepdims=True))
    probs = (probs / probs.sum(1, keepdims=True)).astype(np.float32)
    clamped = np.where(probs < np.float32(1e-4), np.float32(1e-4), probs)
    q64, bar = truth(np.ascontiguousarray(np.transpose(clamped, (0, 2, 3, 1))))
    eng = api.Engine(B, H, W, M)
    d_im = torch.from_numpy(image).cuda()
    labels = np.zeros((B, M), np.float32)
    labels[:, [0, 3]] = 1
    cues = np.zeros((B, M, H, W), np.float32)
    for n in MF64_ITERS:
        p = api.CrfParams.from_buffer_copy(params)
        p.n_iters = n
        d_p = torch.from_numpy(probs).cuda()
        seeds, crf_out = torch.empty_like(d_p), torch.empty_like(d_p)
        eng.dsrg_forward_dev(torch.from_numpy(labels).cuda(), d_p, torch.from_numpy(cues).cuda(), d_im, p, 0.99, 0.85,
                             seeds, crf_out=crf_out)
        check(name + " dsrg_forward_dev", "entry", np.transpose(crf_out.cpu().numpy(), (0, 2, 3, 1)), q64, bar, n,
              range(B))
        d_p = torch.from_numpy(probs).cuda()
        log_out = torch.empty_like(d_p)
        eng.crflayer_forward_dev(d_p, d_im, p, log_out)
        torch.cuda.synchronize()
        check(name + " crflayer_forward_dev", "entry", np.transpose(eng.crf_last_marginals_host(B), (0, 2, 3, 1)),
              q64, bar, n, range(B))
    eng.close()
    # a DenseCRF object on one image, against the float64 bar, the oracle object and the reference build's own
    un = log_unary(1, H, W, M, seed=12)
    q64, bar = Truth(image[:1], params, [0])(un)
    ours, ora = api.DenseCRF(W, H, M), crf_oracle.DenseCRF(W, H, M)
    objs = [ours, ora] + ([crf_oracle.RefDenseCRF(W, H, M)] if crf_oracle.ref_crf_available() else [])
    for c in objs:
        c.set_unary_energy(-un[0].ravel())
        c.add_pairwise_energy(*pairwise_args(params), image[0].ravel())
    for n in MF64_ITERS:
        check(name + " DenseCRF", "entry", ours.inference(n).reshape(1, H, W, M), q64, bar, n, [0])
    want = ora.inference(10).reshape(H, W, M)
    top2 = np.sort(want, -1)[..., -2:]
    bad = ours.map(10).reshape(H, W) != ora.map(10).reshape(H, W)
    assert ((top2[..., 1] - top2[..., 0])[bad] <= 4 * TOL).all()
    if len(objs) > 2:
        got = ours.inference(10).reshape(H, W, M)
        assert np.abs(got - objs[2].inference(10).reshape(H, W, M)).max() <= TOL
    # predict_mask_dev: the scores at the image's size (a zoom by 1), softmax, clamp, CRF with the set's parameters
    one = api.Engine(1, H, W, M)
    scores = torch.from_numpy((rng.randn(M, H, W) * 3).astype(np.float32)).cuda()
    d_im0 = torch.from_numpy(image[0]).cuda()
    res = torch.empty((H, W), dtype=torch.int32, device="cuda")
    soft, crf = torch.empty((H, W, M), device="cuda"), torch.empty((H, W, M), device="cuda")
    one.predict_mask_dev([scores], d_im0, res, params, smooth=False, probs_out=soft)
    one.predict_mask_dev([scores], d_im0, res, params, smooth=True, probs_out=crf)
    torch.cuda.synchronize()
    o = crf_oracle.DenseCRF(W, H, M)
    o.set_unary_energy(-np.log(soft.cpu().numpy()).ravel())
    o.add_pairwise_energy(*pairwise_args(params), image[0].ravel())
    want = o.inference(params.n_iters).reshape(H, W, M)
    assert np.abs(crf.cpu().numpy() - want).max() <= TOL
    top2 = np.sort(want, -1)[..., -2:]
    bad = res.cpu().numpy() != want.argmax(-1)
    assert ((top2[..., 1] - top2[..., 0])[bad] <= 4 * TOL).all()
    one.close()


def test_key_edge_aniso(torch_cuda):
    """At the strip's edge sigmas both lattices build and match the oracle, and the device's key-range flag stays
    clear (crf_host reads it back).  One float32 step below on either x axis, and either pair with x and y swapped,
    is refused before any launch exactly where the restated api.cu:key_range_ok refuses it; the engine goes on."""
    torch = torch_cuda
    H, W = KEY_EDGE_SHAPE
    B = KEY_EDGE_B
    images = set_images("binary", H, W, B)
    eng = api.Engine(B, H, W, PARAM_M)
    params = edge_params(KEY_EDGE_SP, KEY_EDGE_BI)

    def edge_pass():
        eng.crf_host(np.zeros((B, H, W, PARAM_M), np.float32), images, params)
        return check_lattices(eng, images, params, range(B))

    vs, vb, keys = edge_pass()
    assert keys == KEY_EDGE_MAX_KEY
    LAT_ROWS.append(("key_edge_aniso", "-", blur_branch(H, W, vb), vs, int(vb.min()), int(vb.max()), keys[0], keys[1]))
    down = lambda s: float(np.nextafter(np.float32(s), np.float32(0)))   # noqa: E731
    variants = [(KEY_EDGE_SP, (down(KEY_EDGE_BI[0]),) + KEY_EDGE_BI[1:]),
                ((down(KEY_EDGE_SP[0]), KEY_EDGE_SP[1]), KEY_EDGE_BI),
                (KEY_EDGE_SP[::-1], KEY_EDGE_BI),
                (KEY_EDGE_SP, KEY_EDGE_BI[1::-1] + KEY_EDGE_BI[2:])]
    for k, (sp, bi) in enumerate(variants):
        ok = key_range_ok(sp, H, W) and key_range_ok(bi, H, W)
        assert not ok, k                      # test_crf_params_cpu.py pins these claims
        eng.take_launch_count()
        un = torch.zeros((B, H, W, PARAM_M), device="cuda")
        with pytest.raises(_lib.DsrgError) as ei:
            eng.crf_dev(un, torch.from_numpy(images).cuda(), edge_params(sp, bi), torch.empty_like(un))
        assert ei.value.code == _lib.E_KEYRANGE, k
        assert eng.take_launch_count() == 0, k
        for which in (0, 1):
            assert eng.lattice_idle(which) == (0, 0, 0)
        assert edge_pass()[2] == KEY_EDGE_MAX_KEY, k
    eng.close()


FIELDS = ("w1", "theta_alpha_x", "theta_alpha_y", "theta_beta_r", "theta_beta_g", "theta_beta_b", "w2",
          "theta_gamma_x", "theta_gamma_y")
CACHE_BASE = (10, 50, 120, 7, 13, 31, 3, 2, 5)
CACHE_CHANGES = (4.5, 70, 90, 10, 20, 25, -1.5, 3, 4)   # the new value of each field in turn


def cache_steps():
    """(label, nine values, n_iters, calls): the base set, then each field changed in turn, the theta_gamma x <-> y
    swap, n_iters, and a return to the base set."""
    v, n = list(CACHE_BASE), 5
    steps = [("base", tuple(v), n, 2)]
    for field, x in zip(FIELDS, CACHE_CHANGES):
        v[FIELDS.index(field)] = x
        steps.append((field, tuple(v), n, 2))
    v[7], v[8] = v[8], v[7]
    steps.append(("theta_gamma x<->y", tuple(v), n, 2))
    steps.append(("n_iters", tuple(v), 10, 2))
    steps.append(("return to base", CACHE_BASE, 5, 3))
    return steps


def test_cache_and_graph_replay(torch_cuda):
    """One engine with graphs on, on a side stream with the same tensors every call, walks cache_steps.  After every
    call its output matches a fresh graphs-off engine, both lattices match the oracle's for the current values (a
    stale spatial lattice or a replayed build with old sigmas fails here), and the graph-replay counter moves exactly
    when the pass's key (the values, n_iters and whether the spatial lattice is rebuilt) was seen before."""
    torch = torch_cuda
    image = set_images("smooth", 37, 53, 2)
    B, H, W = image.shape[:3]
    M = PARAM_M
    unary = log_unary(B, H, W, M, seed=41)
    eng = api.Engine(B, H, W, M)
    eng.set_graphs(True)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        d_im = torch.from_numpy(image).cuda()
        d_un = torch.from_numpy(unary).cuda()
        out = torch.empty_like(d_un)
    seen, gamma, replays = set(), None, 0
    for label, values, n, calls in cache_steps():
        params = make_params(values, n)
        fresh = api.Engine(B, H, W, M)
        fresh.set_graphs(False)
        want = fresh.crf_host(unary, image, params)
        fresh.close()
        f32 = tuple(float(np.float32(x)) for x in values)
        for call in range(calls):
            rebuild = gamma != f32[7:]
            key = (f32, n, rebuild)
            before = eng.graph_replays
            with torch.cuda.stream(s):
                out.fill_(float("nan"))
                eng.crf_dev(d_un, d_im, params, out, stream=s.cuda_stream)
            s.synchronize()
            assert eng.graph_replays - before == (key in seen), (label, call)
            replays += key in seen
            seen.add(key)
            gamma = f32[7:]
            assert np.abs(out.cpu().numpy() - want).max() <= TOL, (label, call)
            check_lattices(eng, image, params, range(B))
    assert replays >= 10
    eng.close()
