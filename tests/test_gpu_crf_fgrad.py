"""The device's gradient to caller-given bilateral features (dsrg_crf_forward_train_feat_dev,
dsrg_crf_backward_feat_dev, nn.dense_crf(features_bi=...)) against the float64 derivative of
oracle/crf_fgrad_oracle.py, under tests/crf_fgrad_cases.FgradTruth's per-case bars.

Cases: the image path's own features (the lattice tables bit for bit, the marginals, and the identity
sum f . dL/df = dL/dp against the kernel-bandwidth backward), random and learned-looking features on every tile path
of the fused kernels, M in {1, 2, 6, 21, 24, 32}, T in {0, 1, 10}, Potts from the host and the device and matrices,
train-s's batch (20 @ 41x41, 21 labels, 10 iterations) and the benchmark's (64 @ 321x321 photos, hybrid tiles);
FULL_KERNEL (f = P @ raw) through autograd; the unary / Potts / compat gradients against the existing backward; the
per-image NaN policy and its flags; a captured step replayed with new features; an intervening pass, the 33-label
refusal and nn.dense_crf under autocast."""
import numpy as np
import pytest

import helpers
from crf_compat_cases import compat_mats
from crf_fgrad_cases import FgradTruth, case, features_of, inputs
from crf_grad_cases import grad_params
from dsrg_b200 import _lib, api

pytestmark = pytest.mark.gpu

LABELS = (1, 2, 6, 21, 24, 32)
ITERS = (0, 1, 10)


def _nchw(torch, a):
    return torch.from_numpy(np.ascontiguousarray(np.transpose(a, (0, 3, 1, 2)))).cuda()


def _run_feat(torch, eng, feats, unary, G, p, mus=None, potts=None, theta_sp=True):
    """-> dict of the feature entry points' outputs as numpy: q (B, M, H, W), gu, gf (B, 5, H, W), gw, gsp."""
    B, M = unary.shape[0], unary.shape[-1]
    u, g, f = _nchw(torch, unary), _nchw(torch, G), _nchw(torch, feats)
    q_hist = torch.empty((p.n_iters + 1,) + tuple(u.shape), device="cuda")
    gu, gf = torch.empty_like(u), torch.full_like(f, float("nan"))
    gsp = torch.full((B, 2), float("nan"), device="cuda") if theta_sp else None
    if mus is not None:
        compat = torch.from_numpy(np.stack(mus).astype(np.float32)).cuda()
        gw = torch.empty((B, 2, M, M), device="cuda")
        eng.crf_forward_train_feat_dev(u, f, p, q_hist, compat=compat)
        eng.crf_backward_feat_dev(q_hist, f, p, g, gu, gf, compat=compat, grad_compat=gw, grad_theta_sp=gsp)
    else:
        gw = torch.empty((B, 2), device="cuda")
        eng.crf_forward_train_feat_dev(u, f, p, q_hist, potts=potts)
        eng.crf_backward_feat_dev(q_hist, f, p, g, gu, gf, potts=potts, grad_potts=gw, grad_theta_sp=gsp)
    torch.cuda.synchronize()
    out = dict(q=q_hist[-1].cpu().numpy(), gu=gu.cpu().numpy(), gf=gf.cpu().numpy(), gw=gw.cpu().numpy())
    out["gsp"] = gsp.cpu().numpy() if gsp is not None else None
    return out


def _run_image(torch, eng, images, unary, G, p, mus=None):
    """The kernel-bandwidth backward on the image: -> q, gu, gt (B, 7), gw."""
    B, M = unary.shape[0], unary.shape[-1]
    u, g, im = _nchw(torch, unary), _nchw(torch, G), torch.from_numpy(images).cuda()
    q_hist = torch.empty((p.n_iters + 1,) + tuple(u.shape), device="cuda")
    gu, gt = torch.empty_like(u), torch.empty((B, 7), device="cuda")
    if mus is not None:
        compat = torch.from_numpy(np.stack(mus).astype(np.float32)).cuda()
        gw = torch.empty((B, 2, M, M), device="cuda")
        eng.crf_forward_train_compat_dev(u, im, p, compat, q_hist)
        eng.crf_backward_compat_theta_dev(q_hist, im, p, compat, g, gu, gt, grad_compat=gw)
    else:
        gw = torch.empty((B, 2), device="cuda")
        eng.crf_forward_train_dev(u, im, p, q_hist)
        eng.crf_backward_theta_dev(q_hist, im, p, g, gu, gt, grad_potts=gw)
    torch.cuda.synchronize()
    return dict(q=q_hist[-1].cpu().numpy(), gu=gu.cpu().numpy(), gt=gt.cpu().numpy(), gw=gw.cpu().numpy())


def _check_identity(feats, gf, gt, p):
    """sum over the pixels of f . dL/df against the image path's dL/dp = -theta * dL/dtheta, per image and channel,
    within 1e-4 of sum |f . dL/df| (the device adds the same float32 products in another order)."""
    theta = np.array([p.theta_alpha_x, p.theta_alpha_y, p.theta_beta_r, p.theta_beta_g, p.theta_beta_b])
    prod = np.einsum("bchw,bhwc->bchw", gf.astype(np.float64), feats.astype(np.float64))
    dp = prod.reshape(prod.shape[0], 5, -1).sum(2)
    scale = np.abs(prod).reshape(prod.shape[0], 5, -1).sum(2)
    want_dp = -theta[None, :] * gt[:, :5].astype(np.float64)
    assert np.all(np.abs(dp - want_dp) <= 1e-4 * scale + 1e-12), (dp, want_dp, scale)


def _check(got, feats, p, unary, G, mus, compare):
    for b in compare:
        FgradTruth(feats[b], p, unary[b], G[b], mus).check(got["gf"][b], got["gsp"][b], "image %d:" % b)


def _run_case(torch, c, compare=(1,), potts=None):
    images, feats, p, unary, G, mus = c
    B, H, W = images.shape[:3]
    eng = api.Engine(B, H, W, unary.shape[-1])
    got = _run_feat(torch, eng, feats, unary, G, p, mus, potts)
    eng.close()
    _check(got, feats, p, unary, G, mus, compare)
    return got


def sm_count(torch):
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


@pytest.mark.parametrize("img,sf", helpers.FUSED_CONFIGS)
def test_image_features_build_the_image_lattice(torch_cuda, img, sf):
    """features = float32(x)/theta_alpha, ...: offsets, neighbours and barycentric weights equal the image path's."""
    torch = torch_cuda
    images = helpers.fused_images(img)
    B, H, W = images.shape[:3]
    M, p = 6, grad_params(sf, 2)
    feats = np.stack([features_of("image", images[b], p, 0) for b in range(B)])
    unary, G = inputs(B, H, W, M, 10)
    eng = api.Engine(B, H, W, M)
    want = _run_image(torch, eng, images, unary, G, p)
    tables = [(eng.lattice_tables(1, b), eng.lattice_bary(1, b)) for b in range(B)]
    got = _run_feat(torch, eng, feats, unary, G, p)
    for b in range(B):
        (off, nbr), bary = eng.lattice_tables(1, b), eng.lattice_bary(1, b)
        assert np.array_equal(off, tables[b][0][0]) and np.array_equal(nbr, tables[b][0][1])
        assert np.array_equal(bary, tables[b][1])
    assert eng.feature_range_flags(B).tolist() == [False] * B
    eng.close()
    # the same kernels on the same tables: only the order of the float atomics in the splats may differ
    np.testing.assert_allclose(got["q"], want["q"], rtol=0, atol=1e-5)
    np.testing.assert_allclose(got["gu"], want["gu"], rtol=0, atol=1e-4 * float(np.abs(want["gu"]).max()))
    np.testing.assert_allclose(got["gw"], want["gw"], rtol=1e-3, atol=1e-4 * float(np.abs(want["gw"]).max()))
    np.testing.assert_allclose(got["gsp"], want["gt"][:, 5:7], rtol=1e-3, atol=1e-4 * float(np.abs(want["gt"]).max()))
    _check_identity(feats, got["gf"], want["gt"], p)


@pytest.mark.parametrize("path,kind", [("smem", "image"), ("bi_direct", "image"), ("sp_direct", "image"),
                                       ("smem", "guide"), ("bi_direct", "random"), ("sp_direct", "guide")])
def test_feature_gradient_on_every_tile_path(torch_cuda, path, kind):
    img, sf = helpers.MF64_PATH_CONFIG[path]
    c = case(img, sf, kind, 6, 3, seed=11)
    if kind == "image":
        pred = helpers.predict_tile_paths(c[0], sf, sm_count(torch_cuda))
        want = {"smem": ("bi", "smem"), "bi_direct": ("bi", "direct"), "sp_direct": ("sp", "direct")}[path]
        assert (np.asarray(pred[want[0]]) == want[1]).any(), "the case does not reach %s" % path
    _run_case(torch_cuda, c)


@pytest.mark.parametrize("M", LABELS)
@pytest.mark.parametrize("T", ITERS)
def test_feature_gradient_labels_and_iterations(torch_cuda, M, T):
    if T == 10 and M not in (2, 21):
        pytest.skip("ten iterations at two label counts")
    got = _run_case(torch_cuda, case("noise", 1.0, "random", M, T, H=13, W=17, seed=M + T), compare=(0, 1))
    if T == 0 or M == 1:
        assert not np.any(got["gf"]) and not np.any(got["gsp"])


@pytest.mark.parametrize("weights", ["potts_dev", "nonsym", "sym"])
def test_feature_gradient_with_device_weights_and_matrices(torch_cuda, weights):
    torch = torch_cuda
    images, feats, p, unary, G, _ = case("photo", 1.0, "guide", 6, 3, H=19, W=23, seed=5)
    if weights == "potts_dev":
        p.w1, p.w2 = 7.0, 2.0      # the kernels read the device's {w1, w2}; params' own must not leak in
        potts = torch.tensor([4.0, 5.0], device="cuda")
        pt = grad_params(1.0, 3, w1=4.0, w2=5.0)
        got = _run_feat(torch, api.Engine(2, 19, 23, 6), feats, unary, G, p, potts=potts)
        _check(got, feats, pt, unary, G, None, (0, 1))
    else:
        _run_case(torch, (images, feats, p, unary, G, compat_mats(weights, 6, 9)), compare=(0, 1))


@pytest.mark.parametrize("mu", [None, "nonsym"])
def test_other_gradients_match_the_existing_backward(torch_cuda, mu):
    """With the image's own features, grad_unary and grad_potts / grad_compat equal dsrg_crf_backward_dev's /
    dsrg_crf_backward_compat_dev's, and leaving grad_theta_sp out changes nothing."""
    torch = torch_cuda
    images = helpers.fused_images("noise")
    B, H, W = images.shape[:3]
    M, p = 21, grad_params(1.0, 3)
    feats = np.stack([features_of("image", images[b], p, 0) for b in range(B)])
    unary, G = inputs(B, H, W, M, 8)
    mus = compat_mats(mu, M, 5) if mu else None
    eng = api.Engine(B, H, W, M)
    a = _run_feat(torch, eng, feats, unary, G, p, mus)
    b = _run_feat(torch, eng, feats, unary, G, p, mus, theta_sp=False)
    u, g, im = _nchw(torch, unary), _nchw(torch, G), torch.from_numpy(images).cuda()
    q_hist = torch.empty((p.n_iters + 1,) + tuple(u.shape), device="cuda")
    gu = torch.empty_like(u)
    if mus is not None:
        compat = torch.from_numpy(np.stack(mus).astype(np.float32)).cuda()
        gw = torch.empty((B, 2, M, M), device="cuda")
        eng.crf_forward_train_compat_dev(u, im, p, compat, q_hist)
        eng.crf_backward_compat_dev(q_hist, im, p, compat, g, gu, grad_compat=gw)
    else:
        gw = torch.empty((B, 2), device="cuda")
        eng.crf_forward_train_dev(u, im, p, q_hist)
        eng.crf_backward_dev(q_hist, im, p, g, gu, grad_potts=gw)
    torch.cuda.synchronize()
    eng.close()
    # the same kernels; only the order of the float atomics in the splats differs between two runs
    for k in ("q", "gu", "gf", "gw"):
        np.testing.assert_allclose(a[k], b[k], rtol=0, atol=1e-4 * float(np.abs(a[k]).max()) + 1e-7)
    np.testing.assert_allclose(a["gu"], gu.cpu().numpy(), rtol=0, atol=1e-4 * float(np.abs(a["gu"]).max()))
    np.testing.assert_allclose(a["gw"], gw.cpu().numpy(), rtol=1e-3, atol=1e-4 * float(np.abs(a["gw"]).max()))


def test_train_s_batch(torch_cuda):
    """train-s's CRF: 20 images of 41x41, 21 labels, sf 12, 10 iterations; images 0 and 13 against the truth."""
    torch = torch_cuda
    B, H, W, M = 20, 41, 41, 21
    images = np.stack([helpers.small_image(np.random.RandomState(900 + b), H, W, ("noise", "smooth", "photo")[b % 3])
                       for b in range(B)])
    p = grad_params(12.0, 10)
    feats = np.stack([features_of(("guide", "image", "random")[b % 3], images[b], p, b) for b in range(B)])
    unary, G = inputs(B, H, W, M, 910)
    eng = api.Engine(B, H, W, M)
    got = _run_feat(torch, eng, feats, unary, G, p)
    eng.close()
    assert np.all(np.isfinite(got["gf"]))
    _check(got, feats, p, unary, G, None, (0, 13))


def test_benchmark_batch_identity(torch_cuda):
    """64 photos of 321x321 (hybrid tiles) with the image's own features: sum f . dL/df against the kernel-bandwidth
    backward's dL/dp, image by image."""
    torch = torch_cuda
    from dsrg_b200 import synth
    B, H, W, M = 64, 321, 321, 21
    images = np.stack([synth.make_image(np.random.RandomState(950 + b), H, W, "photo") for b in range(B)])
    p = grad_params(1.0, 10)
    feats = np.stack([features_of("image", images[b], p, 0) for b in range(B)])
    unary, G = inputs(B, H, W, M, 960)
    eng = api.Engine(B, H, W, M)
    want = _run_image(torch, eng, images, unary, G, p)
    assert eng.hybrid_tiles > 0
    got = _run_feat(torch, eng, feats, unary, G, p)
    eng.close()
    np.testing.assert_allclose(got["q"], want["q"], rtol=0, atol=1e-5)
    np.testing.assert_allclose(got["gsp"], want["gt"][:, 5:7], rtol=1e-3, atol=1e-4 * float(np.abs(want["gt"]).max()))
    _check_identity(feats, got["gf"], want["gt"], p)


def test_full_kernel_through_autograd(torch_cuda):
    """The reference's FULL_KERNEL: f = P @ raw with raw = (x, y, r, g, b); dL/dP = sum over pixels of dL/df raw^T."""
    torch = torch_cuda
    from dsrg_b200 import nn
    images = helpers.fused_images("smooth")
    B, H, W = images.shape[:3]
    M, T = 6, 3
    p = api.crf_params(1.0, 13, T)
    unary, G = inputs(B, H, W, M, 20)
    y, x = np.mgrid[0:H, 0:W]
    raw = np.stack([np.concatenate([x[..., None], y[..., None], images[b].astype(np.float64)], 2)
                    for b in range(B)]).astype(np.float32)                         # (B, H, W, 5)
    P0 = np.diag(1.0 / np.array([p.theta_alpha_x, p.theta_alpha_y, p.theta_beta_r, p.theta_beta_g, p.theta_beta_b]))
    P0 = P0 + 0.002 * np.random.RandomState(2).randn(5, 5)
    P = torch.tensor(P0, dtype=torch.float32, device="cuda", requires_grad=True)
    rt = _nchw(torch, raw)
    f = torch.einsum("ij,bjhw->bihw", P, rt)
    q = nn.dense_crf(_nchw(torch, unary), None, 1.0, 13, T, features_bi=f)
    (q * _nchw(torch, G)).sum().backward()
    fv = np.transpose(f.detach().cpu().numpy(), (0, 2, 3, 1))
    want, bar = np.zeros((5, 5)), np.zeros((5, 5))
    for b in range(B):
        t = FgradTruth(fv[b], grad_params(1.0, T), unary[b], G[b])
        r = raw[b].reshape(-1, 5).astype(np.float64)
        want += t.want.T @ r
        bar += t.bar[:, None] * np.abs(r).sum(0)[None, :]
    got = P.grad.cpu().numpy()
    assert np.all(np.abs(got - want) <= bar + 1e-4 * np.abs(want).max()), (got, want, bar)


def test_out_of_range_features_give_nan_for_that_image_only(torch_cuda):
    torch = torch_cuda
    images, feats, p, unary, G, _ = case("noise", 1.0, "random", 6, 3, H=13, W=17, seed=30)
    bad = feats.copy()
    bad[1, 3, 4, 0] = 1000.0                       # one pixel of image 1 far outside +-150
    eng = api.Engine(2, 13, 17, 6)
    got = _run_feat(torch, eng, bad, unary, G, p)
    assert eng.feature_range_flags(2).tolist() == [False, True]
    for k in ("q", "gu", "gf", "gw", "gsp"):
        assert np.all(np.isnan(got[k][1])), k
        assert np.all(np.isfinite(got[k][0])), k
    alone = _run_feat(torch, eng, feats, unary, G, p)
    assert eng.feature_range_flags(2).tolist() == [False, False]
    eng.close()
    np.testing.assert_allclose(got["gf"][0], alone["gf"][0], rtol=0, atol=1e-4 * float(np.abs(alone["gf"][0]).max()))
    with pytest.raises(api.DsrgError):            # the flags name the last feature pass's batch only
        eng2 = api.Engine(2, 13, 17, 6)
        try:
            eng2.feature_range_flags(2)
        finally:
            eng2.close()


def test_captured_step_replays_with_new_features(torch_cuda):
    torch = torch_cuda
    from dsrg_b200 import nn
    images, feats, p, unary, G, _ = case("noise", 1.0, "guide", 6, 3, H=19, W=23, seed=40)
    feats2 = np.stack([features_of("random", images[b], p, 77 + b) for b in range(2)])
    u, g = _nchw(torch, unary), _nchw(torch, G)
    w1 = torch.tensor(10.0, device="cuda", requires_grad=True)
    f_static = _nchw(torch, feats).requires_grad_(True)

    def step():
        w1.grad = None
        f_static.grad = None
        q = nn.dense_crf(u, None, 1.0, 13, 3, w1=w1, features_bi=f_static)
        (q * g).sum().backward()
        return q

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        q_out = step()
        gf_out, gw_out = f_static.grad, w1.grad
    with torch.no_grad():
        f_static.copy_(_nchw(torch, feats2))
    graph.replay()
    torch.cuda.synchronize()
    got_q, got_gf, got_gw = q_out.detach().cpu().numpy(), gf_out.cpu().numpy(), float(gw_out)
    eager_f = _nchw(torch, feats2).requires_grad_(True)
    w1e = torch.tensor(10.0, device="cuda", requires_grad=True)
    q = nn.dense_crf(u, None, 1.0, 13, 3, w1=w1e, features_bi=eager_f)
    (q * g).sum().backward()
    np.testing.assert_allclose(got_q, q.detach().cpu().numpy(), rtol=0, atol=1e-5)
    gf = eager_f.grad.cpu().numpy()
    np.testing.assert_allclose(got_gf, gf, rtol=0, atol=1e-4 * float(np.abs(gf).max()))
    assert abs(got_gw - float(w1e.grad)) <= 1e-3 * abs(float(w1e.grad)) + 1e-6


@pytest.mark.parametrize("graphs", [0, 1])
def test_an_intervening_pass(torch_cuda, graphs):
    torch = torch_cuda
    images, feats, p, unary, G, _ = case("smooth", 1.0, "guide", 6, 2, seed=50)
    B, H, W = images.shape[:3]
    eng = api.Engine(B, H, W, 6)
    _lib.lib().dsrg_engine_set_graphs(eng.h, graphs)
    u, g, f = _nchw(torch, unary), _nchw(torch, G), _nchw(torch, feats)
    outs = []
    for _ in range(2):
        q_hist = torch.empty((3,) + tuple(u.shape), device="cuda")
        gu, gf = torch.empty_like(u), torch.empty_like(f)
        eng.crf_forward_train_feat_dev(u, f, p, q_hist)
        # another pass with other sigmas on the same engine before the backward
        out = torch.empty_like(u)
        eng.crf_dev(u, torch.from_numpy(images).cuda(), api.crf_params(12.0), out, unary_layout=api.LAYOUT_NCHW,
                    out_layout=api.LAYOUT_NCHW)
        eng.crf_backward_feat_dev(q_hist, f, p, g, gu, gf, grad_theta_sp=torch.empty((B, 2), device="cuda"))
        torch.cuda.synchronize()
        outs.append(dict(q=q_hist[-1].cpu().numpy(), gf=gf.cpu().numpy(), gsp=np.zeros((B, 2))))
    eng.close()
    _check(dict(gf=outs[1]["gf"], gsp=[None, None]), feats, p, unary, G, None, (0, 1))
    np.testing.assert_allclose(outs[0]["gf"], outs[1]["gf"], rtol=0, atol=1e-4 * float(np.abs(outs[0]["gf"]).max()))


def test_refusals(torch_cuda):
    torch = torch_cuda
    H, W, M = 9, 11, 3
    p = grad_params(1.0, 2)
    eng = api.Engine(2, H, W, M)
    u = torch.zeros((2, M, H, W), device="cuda")
    f = torch.zeros((2, 5, H, W), device="cuda")
    q = torch.zeros((3, 2, M, H, W), device="cuda")
    potts = torch.ones(2, device="cuda")
    compat = torch.zeros((2, M, M), device="cuda")
    with pytest.raises(api.DsrgError):     # Potts and matrices together
        eng.crf_forward_train_feat_dev(u, f, p, q, potts=potts, compat=compat)
    with pytest.raises(api.DsrgError):     # grad_compat without matrices
        eng.crf_backward_feat_dev(q, f, p, u, torch.empty_like(u), torch.empty_like(f),
                                  grad_compat=torch.empty((2, 2, M, M), device="cuda"))
    with pytest.raises(api.DsrgError):     # grad_features is required
        eng.crf_backward_feat_dev(q, f, p, u, torch.empty_like(u), None)
    eng.close()
    eng33 = api.Engine(1, H, W, 33)
    u33 = torch.zeros((1, 33, H, W), device="cuda")
    with pytest.raises(api.DsrgError, match="at most 32"):
        eng33.crf_forward_train_feat_dev(u33, f[:1], p, torch.zeros((3, 1, 33, H, W), device="cuda"))
    with pytest.raises(api.DsrgError, match="at most 32"):
        eng33.crf_backward_feat_dev(torch.zeros((3, 1, 33, H, W), device="cuda"), f[:1], p, u33,
                                    torch.empty_like(u33), torch.empty_like(f[:1]))
    eng33.close()


@pytest.mark.parametrize("autocast", [False, True])
@pytest.mark.parametrize("mu", [None, "nonsym"])
def test_dense_crf_with_features(torch_cuda, autocast, mu):
    torch = torch_cuda
    from dsrg_b200 import nn
    images, feats, p, unary, G, _ = case("noise", 1.0, "guide", 6, 3, H=19, W=23, seed=60)
    mus = compat_mats(mu, 6, 3) if mu else None
    kw = {}
    if mus is not None:
        kw = dict(compat_bi=torch.from_numpy(mus[0].astype(np.float32)).cuda(),
                  compat_sp=torch.from_numpy(mus[1].astype(np.float32)).cuda())
    th_sp = torch.tensor([p.theta_gamma_x, p.theta_gamma_y], dtype=torch.float64, requires_grad=True)
    f = _nchw(torch, feats)
    if autocast:
        f = f.half().float()    # exact in half: the features the autocast run gets
        feats = np.transpose(f.cpu().numpy(), (0, 2, 3, 1))
    fin = (f.half() if autocast else f).requires_grad_(True)
    with torch.autocast("cuda", enabled=autocast):
        q = nn.dense_crf(_nchw(torch, unary), None, 1.0, 13, 3, theta_sp=th_sp, features_bi=fin, **kw)
    assert q.dtype == torch.float32
    (q * _nchw(torch, G)).sum().backward()
    assert fin.grad.dtype == fin.dtype and th_sp.grad.dtype == torch.float64
    gf = fin.grad.float().cpu().numpy()
    for b in range(2):
        t = FgradTruth(feats[b], p, unary[b], G[b], mus)
        if autocast:   # the gradient comes back in half: its rounding on top of the bar
            t.bar = t.bar + 2.0 ** -10 * np.abs(t.want).max(0)
        t.check(gf[b], what="image %d:" % b)
