"""The device's mean field after 1, 2, 3 and 10 iterations against the float64 restatement (oracle/meanfield64.py).

Every other CRF test compares with the float32 oracle under 1e-4, the bar ten amplifying iterations need.  Here each
case and each n_iters has its own bar: helpers.BAR_K times the float32 rounding noise of that case after n iterations
(measured on the CPU models of the oracle's and the device's arithmetic), at least helpers.BAR_FLOOR; after one
iteration that is 15 to 100 times tighter than 1e-4 (tests/test_meanfield64_cpu.py prints it per case).

Cases: every fused configuration at one M per MP (shared-memory tiles, direct tiles of both lattices, tail1 and not),
the hybrid-tile batch at one M per MP, gate 2 and both sides of the blur switches, the label-chunked path, four tiny
shapes with 0..3 phantom lanes, and one case per path with w1 = 0 and one with w2 = 0.  Entry points: crf_dev in both
unary layouts everywhere; dsrg_forward_dev (crf_out), crflayer_forward_dev (crf_last_marginals_host) and a DenseCRF
object at one case; the engine's norm vectors against the float64 norms.  The float64 run serves every n_iters and
each image's lattices serve all of its label counts.  Where a batch is large only some of its images are compared.
"""
import numpy as np
import pytest

import helpers
from helpers import (FUSED_CONFIGS, FUSED_ITER_M, GATE2_SEED, GATE2_SHAPE, HYBRID_M, MF64_GATE2_M, MF64_ITERS,
                     MF64_PATH_CONFIG, MF64_TINY, MF64_TINY_M, MF64_TINY_SEED, MF64_WIDE_M, MF64_ZERO_W,
                     MF64_ZERO_W_M, SWITCH_CASES, Truth, crf_both_layouts, fused_images, hybrid_images, log_unary,
                     mf64_problem_params, predict_tile_paths, seeded_images, small_image, wide_images)
from dsrg_b200 import api

pytestmark = pytest.mark.gpu
ROWS = []          # (case, path, n_iters, device error, bar)


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    if not ROWS:
        return
    print("\n%-34s %-10s %3s  %9s  %9s  %5s" % ("case", "path", "n", "dev err", "bar", "ratio"))
    worst = {}
    for case, path, n, err, bar in ROWS:
        print("%-34s %-10s %3d  %9.2e  %9.2e  %5.2f" % (case, path, n, err, bar, err / bar))
        worst[path] = max(worst.get(path, 0.0), err / bar)
    print("worst device error / bar per path: " + ", ".join("%s %.2f" % kv for kv in sorted(worst.items())))


def check(case, path, got, q64, bar, n, images):
    """got (B, H, W, M) device marginals after n iterations; q64 {b: {n: (H, W, M)}} and bar {b: {n: bar}} for the
    compared images, each image against its own bar; the table keeps the image closest to its bar."""
    rows = [(float(np.abs(got[b] - q64[b][n]).max()), bar[b][n]) for b in images]
    err, b_bar = max(rows, key=lambda r: r[0] / r[1])
    ROWS.append((case, path, n, err, b_bar))
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
    return q64, bar


@pytest.mark.parametrize("img,sf", FUSED_CONFIGS)
def test_fused_paths(torch_cuda, img, sf):
    image = fused_images(img)
    B, H, W = image.shape[:3]
    params = mf64_problem_params(sf)
    truth = Truth(image, params, range(B))
    path = {("smooth", 1.0): "smem", ("noise", 1.0): "bi_direct", ("smooth", 12.0): "sp_direct"}[(img, sf)]
    for M in FUSED_ITER_M:
        run_case(torch_cuda, "%s sf%g M%d" % (img, sf, M), path, image,
                 log_unary(B, H, W, M, seed=1000 * FUSED_CONFIGS.index((img, sf)) + M), params, truth)


def test_hybrid_tiles(torch_cuda):
    image = hybrid_images()
    B, H, W = image.shape[:3]
    sms = torch_cuda.cuda.get_device_properties(torch_cuda.cuda.current_device()).multi_processor_count
    pred = predict_tile_paths(image, 1.0, sms)
    params = mf64_problem_params(1.0)
    hy = pred["bi"] == "hybrid"
    b = int(np.argmax(hy.sum(1)))                   # the image with the most hybrid tiles
    truth = Truth(image, params, [b])
    for M in HYBRID_M:
        eng = api.Engine(B, H, W, M)
        run_case(torch_cuda, "hybrid M%d (image %d)" % (M, b), "hybrid", image,
                 log_unary(B, H, W, M, seed=5000 + M), params, truth, eng)
        assert eng.hybrid_tiles == pred["hybrid_tiles"]
        eng.close()


def test_gate2_and_switches(torch_cuda):
    image = seeded_images(*GATE2_SHAPE, ("noise", "noise"), GATE2_SEED)
    B, H, W = image.shape[:3]
    params = mf64_problem_params(1.0)
    truth = Truth(image, params, [0])
    for M in MF64_GATE2_M:
        eng = api.Engine(B, H, W, M)
        run_case(torch_cuda, "gate2 M%d" % M, "gate2", image, log_unary(B, H, W, M, seed=8000 + M), params, truth,
                 eng)
        assert helpers.blur_branch(H, W, eng.lattice_sizes(B)[1]) == "gate2"
        eng.close()
    for name, H, W, kinds, branch in SWITCH_CASES:
        image = seeded_images(H, W, kinds, GATE2_SEED)
        B = image.shape[0]
        eng = api.Engine(B, H, W, 21)
        run_case(torch_cuda, name, branch, image, log_unary(B, H, W, 21, seed=8100 + H + W), params,
                 Truth(image, params, [0]), eng)
        assert helpers.blur_branch(H, W, eng.lattice_sizes(B)[1]) == branch
        eng.close()


def test_wide_path(torch_cuda):
    for img in ("smooth", "noise"):
        image = wide_images(img)
        B, H, W = image.shape[:3]
        params = mf64_problem_params(1.0)
        truth = Truth(image, params, range(B))
        for M in MF64_WIDE_M:
            run_case(torch_cuda, "wide %s M%d" % (img, M), "wide", image,
                     log_unary(B, H, W, M, seed=7100 + M, scale=4.0), params, truth)


def test_tiny_shapes_phantom_lanes(torch_cuda):
    for H, W, img in MF64_TINY:
        image = np.stack([small_image(np.random.RandomState(MF64_TINY_SEED + b), H, W, img) for b in range(2)])
        params = mf64_problem_params(1.0)
        run_case(torch_cuda, "tiny %dx%d" % (H, W), "tiny", image, log_unary(2, H, W, MF64_TINY_M, seed=3), params,
                 Truth(image, params, range(2)))


@pytest.mark.parametrize("path,zero", MF64_ZERO_W)
def test_one_lattice_only(torch_cuda, path, zero):
    M = MF64_ZERO_W_M[path]
    if path == "hybrid":
        image = hybrid_images()
        compare = [0]
    elif path == "wide":
        image = wide_images("noise")
        compare = [0, 1]
    else:
        image = fused_images(MF64_PATH_CONFIG[path][0])
        compare = [0, 1]
    sf = MF64_PATH_CONFIG.get(path, ("", 1.0))[1]
    B, H, W = image.shape[:3]
    params = mf64_problem_params(sf, zero)
    run_case(torch_cuda, "%s %s=0 M%d" % (path, zero, M), path, image, log_unary(B, H, W, M, seed=77), params,
             Truth(image, params, compare))


def test_other_entry_points_and_norms(torch_cuda):
    """dsrg_forward_dev with crf_out and crflayer_forward_dev (unary: the in-place clamped probs), a DenseCRF object
    (unary energy -log p), and the engine's norm vectors, on the bilateral-direct configuration."""
    torch = torch_cuda
    img, sf = MF64_PATH_CONFIG["bi_direct"]
    image = fused_images(img)
    B, H, W = image.shape[:3]
    M = 21
    params = mf64_problem_params(sf)
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
        check("dsrg_forward_dev", "bi_direct", np.transpose(crf_out.cpu().numpy(), (0, 2, 3, 1)), q64, bar, n,
              range(B))
        d_p = torch.from_numpy(probs).cuda()
        log_out = torch.empty_like(d_p)
        eng.crflayer_forward_dev(d_p, d_im, p, log_out)
        torch.cuda.synchronize()
        raw = eng.crf_last_marginals_host(B)
        check("crflayer_forward_dev", "bi_direct", np.transpose(raw, (0, 2, 3, 1)), q64, bar, n, range(B))
    # the engine's norms: the splat of ones adds in atomic order; the bar is the float32 models' own spread
    ns, nb = eng.norms(B)
    for b in range(B):
        P = truth.problems[b]
        n64 = P.norms(np.float64)
        for k, got in ((0, ns), (1, nb[b])):
            spread = max(float(np.abs(P.norms(np.float32, s)[k] - n64[k]).max() / n64[k].max())
                         for s in (None, 1, 2, 3))
            rel = float(np.abs(got - n64[k]).max() / n64[k].max())
            ROWS.append(("norm lattice %d image %d (rel.)" % (k, b), "norms", 0, rel,
                         max(helpers.BAR_K * spread, 2.0 ** -23)))
            assert rel <= max(helpers.BAR_K * spread, 2.0 ** -23), (k, b, rel, spread)
    eng.close()
    # a DenseCRF object, one image
    un = log_unary(1, H, W, M, seed=12)
    t1 = Truth(image[:1], params, [0])
    q64, bar = t1(un)
    c = api.DenseCRF(W, H, M)
    c.set_unary_energy(-un[0].ravel())
    c.add_pairwise_energy(params.w1, params.theta_alpha_x, params.theta_alpha_y, params.theta_beta_r,
                          params.theta_beta_g, params.theta_beta_b, params.w2, params.theta_gamma_x,
                          params.theta_gamma_y, image[0].ravel())
    for n in MF64_ITERS:
        check("DenseCRF", "bi_direct", c.inference(n).reshape(1, H, W, M), q64, bar, n, [0])
