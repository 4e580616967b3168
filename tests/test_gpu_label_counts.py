"""GPU parity over the whole advertised label range (1..255) against the CPU oracles.

The fused mean-field kernels are instantiated per padded label count MP = 4, 8, ..., 32 (meanfield.cu), with a
special last quad when it holds one real label (`tail1`, M = MP - 3); each instantiation has a shared-memory tile
path, a direct path for overflow tiles and a hybrid-tile kernel.  Label counts above 32 run on the label-chunked
path (meanfield_wide.cu).  The float64 renormalisation (common.cuh:numpy_sum) has an n < 8 branch, a block branch
and a split above 128 labels.  Which tile path each case takes is predicted from the oracle's lattices
(helpers.predict_tile_paths); tests/test_label_counts_cpu.py checks that the case table below reaches every path.

Tolerances: CRF marginals 1e-4 max-abs (BASELINE.json north_star), renormalisation and SRG bit-exact, loss layers
those of test_gpu_dropin.py / test_gpu_loss.py.  Every entry point here accepts every M it is run with; the loss
layers refuse M > 32 (DSRG_E_INVALID), which test_gpu_crf.py::test_label_count_limit_is_reported checks.
"""
import numpy as np
import pytest

from helpers import (FUSED_CONFIGS, FUSED_ITER_M, HYBRID_M, MAX_FUSED, RENORM_M, WIDE_M, crf_both_layouts,
                     fused_images, hybrid_images, log_unary, oracle_batch, predict_tile_paths, small_image, wide_images)
from dsrg_b200 import api
from oracle import crf_oracle, loss_oracle, srg_oracle

pytestmark = pytest.mark.gpu
TOL = 1e-4


def assert_close(got, want, what):
    err = float(np.abs(got - want).max())
    assert err <= TOL, (what, err)


@pytest.mark.parametrize("M", range(1, MAX_FUSED + 1))
def test_fused_path_every_label_count(torch_cuda, M):
    """Every M of the fused path on shared-memory tiles (smooth, sf 1), bilateral direct tiles (noise, sf 1) and
    spatial direct tiles (smooth, sf 12), both unary layouts, the arg-max export, and for one M per MP the first /
    middle / last kernel variants alone (n_iters 1 and 2)."""
    torch = torch_cuda
    for ci, (img, sf) in enumerate(FUSED_CONFIGS):
        image = fused_images(img)
        B, H, W = image.shape[:3]
        unary = log_unary(B, H, W, M, seed=1000 * ci + M)
        want = oracle_batch(image, unary, sf)
        eng = api.Engine(B, H, W, M)
        params = api.crf_params(sf)
        nhwc, nchw = crf_both_layouts(torch, eng, unary, image, params)
        assert_close(nhwc, want, (M, img, sf, "NHWC"))
        assert_close(nchw, want, (M, img, sf, "NCHW"))
        lab = torch.empty(B, H, W, dtype=torch.int32, device="cuda")
        eng.crf_map_dev(torch.from_numpy(unary).cuda(), torch.from_numpy(image).cuda(), params, lab)
        lab = lab.cpu().numpy()
        top2 = np.sort(want, -1)[..., -2:] if M > 1 else np.concatenate([np.zeros_like(want), want], -1)
        clear = (top2[..., 1] - top2[..., 0]) > 4 * TOL
        assert np.array_equal(lab[clear], want.argmax(-1)[clear]), (M, img, sf)
        if M in FUSED_ITER_M:
            for n_iters in (1, 2):
                want_n = oracle_batch(image, unary, sf, n_iters)
                nhwc, nchw = crf_both_layouts(torch, eng, unary, image, api.crf_params(sf, maxiter=n_iters))
                assert_close(nhwc, want_n, (M, img, sf, n_iters, "NHWC"))
                assert_close(nchw, want_n, (M, img, sf, n_iters, "NCHW"))
        eng.close()


@pytest.fixture(scope="module")
def hybrid_batch(torch_cuda):
    image = hybrid_images()
    sms = torch_cuda.cuda.get_device_properties(torch_cuda.cuda.current_device()).multi_processor_count
    pred = predict_tile_paths(image, 1.0, sms)
    assert pred["hybrid_tiles"] > 0, "the textured batch no longer makes a hybrid pass on this device"
    return image, pred


@pytest.mark.parametrize("M", HYBRID_M)
def test_hybrid_tiles_every_padded_label_count(torch_cuda, hybrid_batch, M):
    """k_mf_tile_hy at one M per MP on textured 321x321 images, both layouts, and exactly the hybrid tiles that
    tiles.cu's rules give on the oracle's lattices."""
    torch = torch_cuda
    image, pred = hybrid_batch
    B, H, W = image.shape[:3]
    unary = log_unary(B, H, W, M, seed=5000 + M)
    want = oracle_batch(image, unary, 1.0)
    eng = api.Engine(B, H, W, M)
    d_im = torch.from_numpy(image).cuda()
    d_un = torch.from_numpy(unary).cuda()
    d_out = torch.empty_like(d_un)
    eng.crf_dev(d_un, d_im, api.crf_params(1.0), d_out)
    assert eng.hybrid_tiles == pred["hybrid_tiles"]
    assert_close(d_out.cpu().numpy(), want, (M, "NHWC"))
    d_nchw = d_un.permute(0, 3, 1, 2).contiguous()
    d_out2 = torch.empty_like(d_nchw)
    eng.crf_dev(d_nchw, d_im, api.crf_params(1.0), d_out2, api.LAYOUT_NCHW, api.LAYOUT_NCHW)
    assert eng.hybrid_tiles == pred["hybrid_tiles"]
    assert_close(d_out2.permute(0, 2, 3, 1).cpu().numpy(), want, (M, "NCHW"))
    eng.close()


@pytest.mark.parametrize("M", WIDE_M)
def test_wide_path_label_counts(torch_cuda, M):
    """The label-chunked path up to the advertised 255, with and without padding lanes, smooth and noise images,
    sf 1 and 12, both layouts."""
    torch = torch_cuda
    for img in ("smooth", "noise"):
        image = wide_images(img)
        B, H, W = image.shape[:3]
        eng = api.Engine(B, H, W, M)
        for sf in (1.0, 12.0):
            # sharper unaries than the fused cases: at scale 2 some noise cases sit where a one-ulp change of the
            # unary moves the oracle's own marginals by more than the tolerance (the splat's float32 atomics add in
            # another order than the oracle does)
            unary = log_unary(B, H, W, M, seed=7100 + M + int(sf), scale=4.0)
            want = oracle_batch(image, unary, sf)
            nhwc, nchw = crf_both_layouts(torch, eng, unary, image, api.crf_params(sf))
            assert_close(nhwc, want, (M, img, sf, "NHWC"))
            assert_close(nchw, want, (M, img, sf, "NCHW"))
        eng.close()


@pytest.mark.parametrize("M", RENORM_M)
def test_renormalisation_bit_exact(torch_cuda, M):
    """CRFLayer's device pass (pylayers.py:63-88): the input clamped in place, `result` the float64 clamp +
    renormalisation of the raw marginals in NumPy's summation order cast to float32, `log_out` its log; and the SRG
    with that renormalisation fused in (renorm=True) equals the SRG on the renormalised marginals."""
    torch = torch_cuda
    B, H, W = 2, 11, 19
    rng = np.random.RandomState(300 + M)
    logits = rng.randn(B, M, H, W)
    logits[:, 0, : H // 2] += 12          # confident pixels: every other label far below 1e-4
    probs = np.exp(logits - logits.max(1, keepdims=True))
    probs = (probs / probs.sum(1, keepdims=True)).astype(np.float32)
    image = np.stack([small_image(np.random.RandomState(40 + b), H, W, "smooth") for b in range(B)])
    eng = api.Engine(B, H, W, M)
    d_p = torch.from_numpy(probs).cuda()
    log_out, result = torch.empty_like(d_p), torch.empty_like(d_p)
    eng.crflayer_forward_dev(d_p, torch.from_numpy(image).cuda(), api.crf_params(12.0), log_out, result)
    torch.cuda.synchronize()
    floor = np.float32(1e-4)
    assert np.array_equal(d_p.cpu().numpy(), np.where(probs < floor, floor, probs))
    raw = eng.crf_last_marginals_host(B)
    r64 = crf_oracle.renormalise(raw)
    assert np.array_equal(result.cpu().numpy(), r64.astype(np.float32))
    assert np.array_equal(log_out.cpu().numpy(), np.log(r64).astype(np.float32))
    labels = np.zeros((B, M), np.float32)
    labels[:, [0, M - 1]] = 1
    cues = (rng.rand(B, M, H, W) < 0.03).astype(np.float32)
    seeds = eng.srg_host(labels, raw, cues, 0.6, 0.004, renorm=True)
    for b in range(B):
        assert np.array_equal(seeds[b], srg_oracle.srg_closed_form(labels[b], cues[b], r64[b], 0.6, 0.004))
    # The CRF's marginals share one binary exponent at high M, so their float64 sums are exact in any order, and a
    # float32 result hides the last bit of a float64 one.  What the summation order decides is the strict threshold
    # compares of the label map (pylayers.py:251-257).  With raw values over four decades, a tenth of them clamped,
    # every class present and both thresholds at one pixel's renormalised maximum, the oracle leaves that pixel
    # unlabelled; a sum formed in another order that comes out one ulp smaller labels it.
    raw2 = (rng.rand(B, M, H, W) ** 4).astype(np.float32)
    r2 = crf_oracle.renormalise(raw2)
    every = np.ones((B, M), np.float32)
    d_raw = torch.from_numpy(raw2).cuda()
    d_every, d_nocue, out = torch.from_numpy(every).cuda(), torch.zeros_like(d_raw), torch.empty_like(d_raw)
    lm = torch.empty(B, H, W, dtype=torch.int32, device="cuda")
    nocue = np.zeros((M, H, W), np.float32)
    for th in np.unique(r2.max(1)):
        eng.srg_dev(d_every, d_raw, d_nocue, th, th, out, renorm=True, label_map_out=lm)
        got = lm.cpu().numpy()
        for b in range(B):
            assert np.array_equal(got[b], srg_oracle.label_map_closed_form(every[b], nocue, r2[b], th, th)), (th, b)
    eng.close()


@pytest.mark.parametrize("M", [64, 128, 254, 255])
def test_srg_wide_label_counts(torch_cuda, M):
    """SRG at label counts above the fused CRF's: the label map stores c + 1 in a byte, 255 labels fill it."""
    torch = torch_cuda
    B, H, W = 2, 23, 31
    rng = np.random.RandomState(900 + M)
    logits = rng.randn(B, M, H, W)
    for c, (ys, xs) in ((0, (slice(0, 8), slice(None))), (5, (slice(8, 16), slice(0, 15))),
                        (M - 1, (slice(8, None), slice(15, None)))):
        logits[:, c, ys, xs] += 10
    probs = np.exp(logits - logits.max(1, keepdims=True))
    probs = np.ascontiguousarray(probs / probs.sum(1, keepdims=True), np.float32)
    labels = np.zeros((B, M), np.float32)
    labels[:, [0, 5, M - 1]] = 1
    cues = (rng.rand(B, M, H, W) < 0.01).astype(np.float32)
    cues[:, M - 1, 12, 20] = 1
    eng = api.Engine(B, H, W, M)
    seeds = eng.srg_host(labels, probs, cues, 0.9, 0.5)
    out = torch.empty(B, M, H, W, device="cuda")
    lm = torch.empty(B, H, W, dtype=torch.int32, device="cuda")
    eng.srg_dev(torch.from_numpy(labels).cuda(), torch.from_numpy(probs).cuda(), torch.from_numpy(cues).cuda(),
                0.9, 0.5, out, label_map_out=lm)
    torch.cuda.synchronize()
    for b in range(B):
        want, wlm = srg_oracle.srg_closed_form(labels[b], cues[b], probs[b], 0.9, 0.5, return_label_map=True)
        assert wlm.max() == M
        assert np.array_equal(seeds[b], want)
        assert np.array_equal(out[b].cpu().numpy(), want)
        assert np.array_equal(lm[b].cpu().numpy(), wlm)
    eng.close()


@pytest.mark.parametrize("M,B,H,W", [(1, 2, 9, 7), (2, 3, 17, 13), (31, 2, 21, 19), (32, 4, 64, 64)])
def test_softmax_and_constrain_loss_label_counts(torch_cuda, M, B, H, W):
    """SoftmaxLayer / ConstrainLossLayer kernels at other label counts; at 4 x 32 x 64 x 64 the grid-stride loops of
    k_constrain_* run more than one pass."""
    rng = np.random.RandomState(50 + M)
    eng = api.Engine(B, H, W, M)
    x = (rng.randn(B, M, H, W) * 3).astype(np.float32)
    probs = eng.softmax_forward_host(x)
    np.testing.assert_allclose(probs, loss_oracle.softmax_layer_forward(x), rtol=2e-5, atol=1e-9)
    g = rng.randn(*x.shape).astype(np.float32)
    np.testing.assert_allclose(eng.softmax_backward_host(x, g), loss_oracle.softmax_layer_backward(x, g),
                               rtol=2e-4, atol=2e-7)
    logs = np.log(rng.uniform(0.01, 1.0, x.shape)).astype(np.float32)
    want = loss_oracle.constrain_loss(probs, logs)
    assert abs(eng.constrainloss_forward_host(probs, logs) - want) <= 2e-5 * abs(want)
    gp, gl = eng.constrainloss_backward_host(probs, logs)
    wp, wl = loss_oracle.constrain_loss_grad(probs.astype(np.float64), logs.astype(np.float64))
    ratio = np.exp(logs.astype(np.float64)) / probs
    safe = (np.abs(ratio - 0.05) > 1e-5) & (np.abs(ratio - 20) > 1e-3)
    np.testing.assert_allclose(gp[safe], wp[safe], rtol=2e-4, atol=1e-9)
    np.testing.assert_allclose(gl[safe], wl[safe], rtol=2e-4, atol=1e-9)
    eng.close()


@pytest.mark.parametrize("M", [1, 2, 32])
def test_seedloss_label_counts(torch_cuda, M):
    """BalancedSeedLoss at other label counts, with an image that has no foreground seeds."""
    torch = torch_cuda
    B, H, W = 3, 19, 23
    rng = np.random.RandomState(70 + M)
    logits = rng.randn(B, M, H, W) * 2
    probs = np.exp(logits - logits.max(1, keepdims=True))
    probs = (probs / probs.sum(1, keepdims=True)).astype(np.float32)
    probs[probs < 1e-4] = 1e-4
    seeds = (rng.rand(B, M, H, W) < 0.05).astype(np.float32)
    seeds[1, 1:] = 0
    eng = api.Engine(B, H, W, M)
    d_p, d_s = torch.from_numpy(probs).cuda(), torch.from_numpy(seeds).cuda()
    terms = torch.zeros(2, device="cuda")
    eng.seedloss_forward_dev(d_p, d_s, terms)
    loss = -float(terms.sum().item()) / B
    want = loss_oracle.balanced_seed_loss(probs, seeds)
    assert abs(loss - want) <= 1e-5 * abs(want)
    grad = torch.empty_like(d_p)
    eng.seedloss_backward_dev(d_p, d_s, grad)
    np.testing.assert_allclose(grad.cpu().numpy(), loss_oracle.balanced_seed_loss_grad(probs, seeds),
                               rtol=1e-5, atol=1e-9)
    eng.close()
