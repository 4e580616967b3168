"""The kernel-bandwidth and feature gradients above 32 labels (dsrg_crf_backward_wide_theta_dev, the
dsrg_crf_forward_train_wide_feat_dev / dsrg_crf_backward_wide_feat_dev pair, nn.dense_crf_wide(theta_bi=...,
theta_sp=..., features_bi=...)) against the float64 exact derivatives of oracle/crf_kgrad_oracle.py and
oracle/crf_fgrad_oracle.py.

Bars: tests/crf_wide_kgrad_cases.py (the float32 models' error, with a floor re-derived for the label-chunked sums);
test_crf_wide_kgrad_cpu.py shows every oracle mutant outside them on every case here.

Cases: M in {33, 36, 81, 128, 255} and T in {0, 1, 2, 10} at scale factors 1 and 12; smooth, photo and noise images
with host and device Potts weights and a non-symmetric mu; anisotropic and per-channel sigmas; image, guide and random
features.  Cross-checks without an oracle at batch 8 @ 321x321 photo-like with 81 labels: the image's own features
build the image's lattice bit for bit, give the theta path's other gradients, and sum f . dL/df = -theta dL/dtheta.
Runs: two backwards, an inference pass in between, COCO's training shape through autograd, the NaN policy, a captured
feature step, theta refused in capture; the refusals."""
import numpy as np
import pytest

import helpers
from crf_compat_cases import compat_mats
from crf_grad_cases import grad_params
from crf_wide_kgrad_cases import (ANISO_RUNS, FEATURE_RUNS, IMAGE_RUNS, LABEL_RUNS, WideFgradTruth, WideKgradTruth,
                                  aniso_case, feature_case, image_case, inputs, label_case)
from crf_fgrad_cases import features_of
from dsrg_b200 import _lib, api, nn

pytestmark = pytest.mark.gpu


def _nchw(torch, a):
    return torch.from_numpy(np.ascontiguousarray(np.transpose(a, (0, 3, 1, 2)))).cuda()


def _compat(torch, mus):
    return None if mus is None else torch.from_numpy(np.stack(mus).astype(np.float32)).cuda()


def run_theta(torch, eng, images, unary, G, p, mus=None, potts=None, between=None):
    """-> dict q, gu, gt (B, 7), gw from the wide forward and dsrg_crf_backward_wide_theta_dev."""
    B, M = unary.shape[0], unary.shape[-1]
    u, g, im = _nchw(torch, unary), _nchw(torch, G), torch.from_numpy(images).cuda()
    q_hist = torch.empty((p.n_iters + 1,) + tuple(u.shape), device="cuda")
    gu, gt = torch.empty_like(u), torch.full((B, 7), float("nan"), device="cuda")
    compat = _compat(torch, mus)
    gw = torch.empty((B, 2, M, M) if mus is not None else (B, 2), device="cuda")
    eng.crf_forward_train_wide_dev(u, im, p, q_hist, potts=potts, compat=compat)
    if between is not None:
        between(eng)
    eng.crf_backward_wide_theta_dev(q_hist, im, p, g, gu, gt, potts=potts, compat=compat,
                                    grad_potts=None if mus is not None else gw,
                                    grad_compat=gw if mus is not None else None)
    torch.cuda.synchronize()
    return dict(q=q_hist[-1].cpu().numpy(), gu=gu.cpu().numpy(), gt=gt.cpu().numpy(), gw=gw.cpu().numpy())


def run_feat(torch, eng, feats, unary, G, p, mus=None, potts=None):
    """-> dict q, gu, gf (B, 5, H, W), gsp (B, 2), gw from the wide feature pair."""
    B, M = unary.shape[0], unary.shape[-1]
    u, g, f = _nchw(torch, unary), _nchw(torch, G), _nchw(torch, feats)
    q_hist = torch.empty((p.n_iters + 1,) + tuple(u.shape), device="cuda")
    gu, gf = torch.empty_like(u), torch.full_like(f, float("nan"))
    gsp = torch.full((B, 2), float("nan"), device="cuda")
    compat = _compat(torch, mus)
    gw = torch.empty((B, 2, M, M) if mus is not None else (B, 2), device="cuda")
    eng.crf_forward_train_wide_feat_dev(u, f, p, q_hist, potts=potts, compat=compat)
    eng.crf_backward_wide_feat_dev(q_hist, f, p, g, gu, gf, potts=potts, compat=compat,
                                   grad_potts=None if mus is not None else gw,
                                   grad_compat=gw if mus is not None else None, grad_theta_sp=gsp)
    torch.cuda.synchronize()
    return dict(q=q_hist[-1].cpu().numpy(), gu=gu.cpu().numpy(), gf=gf.cpu().numpy(), gsp=gsp.cpu().numpy(),
                gw=gw.cpu().numpy())


def check_theta(images, p, unary, G, mus, got, compare=(0, 1)):
    for b in compare:
        WideKgradTruth(images[b], p, unary[b], G[b], mus).check(got["gt"][b], "image %d:" % b)


def check_feat(feats, p, unary, G, mus, got, compare=(0, 1)):
    for b in compare:
        WideFgradTruth(feats[b], p, unary[b], G[b], mus).check(got["gf"][b], got["gsp"][b], "image %d:" % b)


@pytest.mark.parametrize("M,T,sf", LABEL_RUNS)
def test_theta_labels_and_iterations(torch_cuda, M, T, sf):
    images, p, unary, G, mus = label_case(M, T, sf)
    eng = api.Engine(2, images.shape[1], images.shape[2], M)
    got = run_theta(torch_cuda, eng, images, unary, G, p)
    eng.close()
    if T == 0:
        assert not np.any(got["gt"]), got["gt"]
    check_theta(images, p, unary, G, mus, got)


@pytest.mark.parametrize("img,mu", IMAGE_RUNS)
def test_theta_on_every_image_kind(torch_cuda, img, mu):
    images, p, unary, G, mus = image_case(img, mu)
    potts = torch_cuda.tensor([7.5, 4.0], device="cuda") if mu == "potts_dev" else None
    if potts is not None:
        p.w1, p.w2 = 99.0, -99.0   # the device weights must win
    eng = api.Engine(2, 41, 41, 81)
    got = run_theta(torch_cuda, eng, images, unary, G, p, mus, potts)
    eng.close()
    if potts is not None:
        p.w1, p.w2 = 7.5, 4.0
    check_theta(images, p, unary, G, mus, got)


@pytest.mark.parametrize("name,mu", ANISO_RUNS)
def test_theta_at_anisotropic_sigmas(torch_cuda, name, mu):
    images, p, unary, G, mus = aniso_case(name, mu)
    eng = api.Engine(2, images.shape[1], images.shape[2], 36)
    got = run_theta(torch_cuda, eng, images, unary, G, p, mus)
    eng.close()
    check_theta(images, p, unary, G, mus, got)


@pytest.mark.parametrize("kind,M,T,mu", FEATURE_RUNS)
def test_features(torch_cuda, kind, M, T, mu):
    images, feats, p, unary, G, mus = feature_case(kind, M, T, mu)
    eng = api.Engine(2, images.shape[1], images.shape[2], M)
    got = run_feat(torch_cuda, eng, feats, unary, G, p, mus)
    assert eng.feature_range_flags(2).tolist() == [False, False]
    eng.close()
    if T == 0:
        assert not np.any(got["gf"]) and not np.any(got["gsp"])
    check_feat(feats, p, unary, G, mus, got)


@pytest.fixture(scope="module")
def photo_81(torch_cuda):
    """Batch 8 @ 321x321 photo-like, 81 labels: the theta path, then the image's own features on the same engine."""
    torch = torch_cuda
    from dsrg_b200 import synth
    B, H, W, M = 8, 321, 321, 81
    images = np.stack([synth.make_image(np.random.RandomState(950 + b), H, W, "photo") for b in range(B)])
    p = grad_params(1.0, 3)
    feats = np.stack([features_of("image", images[b], p, 0) for b in range(B)])
    unary, G = inputs(B, H, W, M, 960)
    out = {}
    for mu in (None, "nonsym"):
        mus = compat_mats(mu, M, 9) if mu else None
        eng = api.Engine(B, H, W, M)
        th = run_theta(torch, eng, images, unary, G, p, mus)
        tables = [(eng.lattice_tables(1, b), eng.lattice_bary(1, b)) for b in range(B)]
        ft = run_feat(torch, eng, feats, unary, G, p, mus)
        ftables = [(eng.lattice_tables(1, b), eng.lattice_bary(1, b)) for b in range(B)]
        flags = eng.feature_range_flags(B).tolist()
        eng.close()
        out[mu] = (th, ft, tables, ftables, flags)
    return images, feats, p, out


def test_image_features_build_the_image_lattice_at_321(photo_81):
    for th, ft, tables, ftables, flags in photo_81[3].values():
        assert flags == [False] * len(tables)
        for ((off, nbr), bary), ((foff, fnbr), fbary) in zip(tables, ftables):
            assert np.array_equal(off, foff) and np.array_equal(nbr, fnbr) and np.array_equal(bary, fbary)


def test_image_features_give_the_theta_paths_other_gradients(photo_81):
    """The same kernels on the same tables: only the order of the float atomics in the splats may differ."""
    for th, ft, _, _, _ in photo_81[3].values():
        np.testing.assert_allclose(ft["q"], th["q"], rtol=0, atol=1e-5)
        np.testing.assert_allclose(ft["gu"], th["gu"], rtol=0, atol=1e-4 * float(np.abs(th["gu"]).max()))
        np.testing.assert_allclose(ft["gw"], th["gw"], rtol=1e-3, atol=1e-4 * float(np.abs(th["gw"]).max()))
        np.testing.assert_allclose(ft["gsp"], th["gt"][:, 5:7], rtol=1e-3, atol=1e-4 * float(np.abs(th["gt"]).max()))


def test_feature_identity_at_321(photo_81):
    """sum over the pixels of f . dL/df = -theta * dL/dtheta per image and channel, within 1e-4 of sum |f . dL/df|."""
    _, feats, p, out = photo_81
    theta = np.array([p.theta_alpha_x, p.theta_alpha_y, p.theta_beta_r, p.theta_beta_g, p.theta_beta_b])
    for th, ft, _, _, _ in out.values():
        prod = np.einsum("bchw,bhwc->bchw", ft["gf"].astype(np.float64), feats.astype(np.float64))
        dp = prod.reshape(prod.shape[0], 5, -1).sum(2)
        scale = np.abs(prod).reshape(prod.shape[0], 5, -1).sum(2)
        want = -theta[None, :] * th["gt"][:, :5].astype(np.float64)
        assert np.all(np.abs(dp - want) <= 1e-4 * scale + 1e-12), (dp, want, scale)


@pytest.mark.parametrize("mu", [None, "nonsym"])
def test_two_backwards_agree(torch_cuda, mu):
    """The parameter and per-pixel sums run in a fixed order; what two runs may differ by is the order of the splats'
    float atomics (shared with dsrg_crf_backward_wide_dev), far inside the truth's bar."""
    torch = torch_cuda
    images, feats, p, unary, G, _ = feature_case("guide", 81, 3)
    mus = compat_mats(mu, 81, 9) if mu else None
    eng = api.Engine(2, images.shape[1], images.shape[2], 81)
    a, b = run_theta(torch, eng, images, unary, G, p, mus), run_theta(torch, eng, images, unary, G, p, mus)
    fa, fb = run_feat(torch, eng, feats, unary, G, p, mus), run_feat(torch, eng, feats, unary, G, p, mus)
    eng.close()
    t = WideKgradTruth(images[0], p, unary[0], G[0], mus)
    assert np.all(np.abs(a["gt"][0] - b["gt"][0]) <= 0.25 * t.bar)
    np.testing.assert_allclose(fa["gf"], fb["gf"], rtol=0, atol=1e-5 * float(np.abs(fa["gf"]).max()))
    np.testing.assert_allclose(a["gu"], b["gu"], rtol=0, atol=1e-5 * float(np.abs(a["gu"]).max()))


def test_inference_between_forward_and_backward(torch_cuda):
    torch = torch_cuda
    images, p, unary, G, _ = image_case("smooth", "potts_host")
    other = np.ascontiguousarray(images[::-1])

    def infer(eng):
        u = _nchw(torch, helpers.log_unary(2, 41, 41, 81, 99))
        out = torch.empty_like(u)
        eng.crf_dev(u, torch.from_numpy(other).cuda(), grad_params(1.0, 4), out, unary_layout=api.LAYOUT_NCHW,
                    out_layout=api.LAYOUT_NCHW)

    for mus in (None, compat_mats("nonsym", 81, 1)):
        eng = api.Engine(2, 41, 41, 81)
        got = run_theta(torch, eng, images, unary, G, p, mus, between=infer)
        eng.close()
        check_theta(images, p, unary, G, mus, got)


@pytest.mark.parametrize("what", ["theta", "features"])
def test_coco_training_shape_through_dense_crf_wide(torch_cuda, what):
    """Batch 20 @ 41x41, 81 labels, sf 12, T = 10 through nn.dense_crf_wide's autograd, on four problems repeated over
    the slots: every slot's dL/dunary against the same step on the engine's entry points (dsrg_crf_backward_wide_dev
    for theta, the feature pair for features) and against the slots of the same problem, every slot's dL/df against
    its problem's truth, the parameters' against the batch sum of the truths under the sum of the bars."""
    torch = torch_cuda
    B, H, W, M, T = 20, 41, 41, 81, 10
    k = [b % 4 for b in range(B)]
    kinds = ("noise", "smooth", "photo", "photo")
    images = np.stack([helpers.small_image(np.random.RandomState(900 + i), H, W, kinds[i]) for i in k])
    p = grad_params(12.0, T)
    unary, G = (a[k] for a in inputs(4, H, W, M, 910))
    u, g = _nchw(torch, unary).requires_grad_(True), _nchw(torch, G)
    w1 = torch.tensor(10.0, device="cuda", requires_grad=True)
    if what == "theta":
        th_bi = torch.tensor([p.theta_alpha_x, p.theta_alpha_y, p.theta_beta_r, p.theta_beta_g, p.theta_beta_b],
                             dtype=torch.float64, requires_grad=True)
        th_sp = torch.tensor([p.theta_gamma_x, p.theta_gamma_y], dtype=torch.float64, device="cuda",
                             requires_grad=True)
        out = nn.dense_crf_wide(u, torch.from_numpy(images).cuda(), 12.0, maxiter=T, w1=w1, theta_bi=th_bi,
                                theta_sp=th_sp)
    else:
        fk = ("guide", "image", "random", "guide")
        feats = np.stack([features_of(fk[i], images[b], p, i) for b, i in enumerate(k)])
        f = _nchw(torch, feats).requires_grad_(True)
        th_sp = torch.tensor([p.theta_gamma_x, p.theta_gamma_y], dtype=torch.float64, requires_grad=True)
        out = nn.dense_crf_wide(u, None, 12.0, maxiter=T, w1=w1, theta_sp=th_sp, features_bi=f)
    (out * g).sum().backward()
    torch.cuda.synchronize()
    gu = u.grad.cpu().numpy()
    assert np.all(np.isfinite(gu)) and np.isfinite(float(w1.grad))
    # the same step without autograd, on an engine of its own (Potts weights {w1, CRF()'s w2} on the device)
    eng = api.Engine(B, H, W, M)
    potts = torch.tensor([10.0, 3.0], device="cuda")
    if what == "theta":
        ref = run_theta(torch, eng, images, unary, G, p, potts=potts)
        eng2 = api.Engine(B, H, W, M)   # the backward without the theta gradient
        q_hist = torch.empty((T + 1,) + tuple(u.shape), device="cuda")
        gu_w, gw_w = torch.empty_like(u), torch.empty((B, 2), device="cuda")
        im = torch.from_numpy(images).cuda()
        eng2.crf_forward_train_wide_dev(u.detach(), im, p, q_hist, potts=potts)
        eng2.crf_backward_wide_dev(q_hist, im, p, g, gu_w, potts=potts, grad_potts=gw_w)
        torch.cuda.synchronize()
        eng2.close()
        refs = (ref["gu"], gu_w.cpu().numpy())
        gw_ref = gw_w.cpu().numpy()
    else:
        ref = run_feat(torch, eng, feats, unary, G, p, potts=potts)
        refs, gw_ref = (ref["gu"],), ref["gw"]
    eng.close()
    for b, i in enumerate(k):
        tol = 1e-4 * float(np.abs(gu[b]).max())
        for r in refs:
            np.testing.assert_allclose(gu[b], r[b], rtol=0, atol=tol, err_msg="slot %d" % b)
        np.testing.assert_allclose(gu[b], gu[i], rtol=0, atol=tol, err_msg="slot %d against slot %d" % (b, i))
    assert abs(float(w1.grad) - gw_ref[:, 0].sum()) <= 1e-3 * abs(gw_ref[:, 0]).sum()
    if what == "theta":
        got = np.concatenate([th_bi.grad.numpy(), th_sp.grad.cpu().numpy()])
        truths = [WideKgradTruth(images[i], p, unary[i], G[i]) for i in range(4)]
        want, bar = sum(truths[i].want for i in k), sum(truths[i].bar for i in k)
        assert np.all(np.abs(got - want) <= bar), (got, want, bar)
        assert th_sp.grad.device.type == "cuda" and th_bi.grad.device.type == "cpu"
    else:
        gf = f.grad.cpu().numpy()
        want_sp, bar_sp = np.zeros(2), np.zeros(2)
        truths = [WideFgradTruth(feats[i], p, unary[i], G[i]) for i in range(4)]
        for b, i in enumerate(k):
            truths[i].check(gf[b], None, "slot %d:" % b)
            want_sp += truths[i].want_sp
            bar_sp += truths[i].bar_sp
        assert np.all(np.abs(th_sp.grad.numpy() - want_sp) <= bar_sp), (th_sp.grad, want_sp, bar_sp)


def test_out_of_range_features_give_nan_for_that_image_only(torch_cuda):
    torch = torch_cuda
    images, feats, p, unary, G, _ = feature_case("random", 33, 3)
    bad = feats.copy()
    bad[1, 3, 4, 0] = 1000.0                       # one pixel of image 1 far outside +-150
    eng = api.Engine(2, images.shape[1], images.shape[2], 33)
    got = run_feat(torch, eng, bad, unary, G, p)
    assert eng.feature_range_flags(2).tolist() == [False, True]
    for k in ("q", "gu", "gf", "gw", "gsp"):
        assert np.all(np.isnan(got[k][1])), k
        assert np.all(np.isfinite(got[k][0])), k
    alone = run_feat(torch, eng, feats, unary, G, p)
    assert eng.feature_range_flags(2).tolist() == [False, False]
    eng.close()
    np.testing.assert_allclose(got["gf"][0], alone["gf"][0], rtol=0, atol=1e-4 * float(np.abs(alone["gf"][0]).max()))


def test_captured_feature_step_replays_with_new_features(torch_cuda):
    torch = torch_cuda
    images, feats, p, unary, G, _ = feature_case("guide", 81, 3)
    feats2 = np.stack([features_of("random", images[b], p, 77 + b) for b in range(2)])
    u, g = _nchw(torch, unary), _nchw(torch, G)
    w1 = torch.tensor(10.0, device="cuda", requires_grad=True)
    f_static = _nchw(torch, feats).requires_grad_(True)

    def step():
        w1.grad = None
        f_static.grad = None
        q = nn.dense_crf_wide(u, None, 1.0, 13, 3, w1=w1, features_bi=f_static)
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
    q = nn.dense_crf_wide(u, None, 1.0, 13, 3, w1=w1e, features_bi=eager_f)
    (q * g).sum().backward()
    np.testing.assert_allclose(got_q, q.detach().cpu().numpy(), rtol=0, atol=1e-5)
    gf = eager_f.grad.cpu().numpy()
    np.testing.assert_allclose(got_gf, gf, rtol=0, atol=1e-4 * float(np.abs(gf).max()))
    assert abs(got_gw - float(w1e.grad)) <= 1e-3 * abs(float(w1e.grad)) + 1e-6


@pytest.mark.parametrize("where", ["cpu", "cuda"])
def test_theta_refused_in_capture(torch_cuda, where):
    torch = torch_cuda
    u = torch.zeros((1, 40, 9, 11), device="cuda")
    im = torch.zeros((1, 9, 11, 3), dtype=torch.uint8, device="cuda")
    th = torch.ones(2, device=where)
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        g.capture_begin()
        try:
            with pytest.raises(ValueError, match="capture"):
                nn.dense_crf_wide(u, im, theta_sp=th)
        finally:
            g.capture_end()


def test_autocast_casts_the_features(torch_cuda):
    torch = torch_cuda
    images, feats, p, unary, G, _ = feature_case("guide", 33, 2)
    u, g, f = _nchw(torch, unary), _nchw(torch, G), _nchw(torch, feats)
    want = nn.dense_crf_wide(u, None, 1.0, 13, 2, features_bi=f)
    with torch.autocast("cuda", dtype=torch.float16):
        got = nn.dense_crf_wide(u.half(), None, 1.0, 13, 2, features_bi=f.half())
    assert got.dtype == torch.float32
    fh = f.half().float()
    want_h = nn.dense_crf_wide(u.half().float(), None, 1.0, 13, 2, features_bi=fh)
    torch.testing.assert_close(got, want_h, rtol=0, atol=1e-5)
    assert want.shape == got.shape


def test_refusals(torch_cuda):
    torch = torch_cuda
    H, W = 9, 11
    p = grad_params(1.0, 2)
    im = torch.zeros((2, H, W, 3), dtype=torch.uint8, device="cuda")
    for M in (21, 32):   # the label-chunked entry points refuse what the fused ones serve
        eng = api.Engine(2, H, W, M)
        u = torch.zeros((2, M, H, W), device="cuda")
        f = torch.zeros((2, 5, H, W), device="cuda")
        q = torch.zeros((3, 2, M, H, W), device="cuda")
        eng.take_launch_count()
        for call in (lambda: eng.crf_backward_wide_theta_dev(q, im, p, u, torch.empty_like(u),
                                                             torch.empty((2, 7), device="cuda")),
                     lambda: eng.crf_forward_train_wide_feat_dev(u, f, p, q),
                     lambda: eng.crf_backward_wide_feat_dev(q, f, p, u, torch.empty_like(u), torch.empty_like(f))):
            with pytest.raises(api.DsrgError) as e:
                call()
            assert e.value.code == _lib.E_INVALID
        assert eng.take_launch_count() == 0
        eng.close()
    eng = api.Engine(2, H, W, 40)
    u = torch.zeros((2, 40, H, W), device="cuda")
    f = torch.zeros((2, 5, H, W), device="cuda")
    q = torch.zeros((3, 2, 40, H, W), device="cuda")
    eng.take_launch_count()
    with pytest.raises(api.DsrgError):     # grad_theta is required
        eng.crf_backward_wide_theta_dev(q, im, p, u, torch.empty_like(u), None)
    with pytest.raises(api.DsrgError):     # grad_features is required
        eng.crf_backward_wide_feat_dev(q, f, p, u, torch.empty_like(u), None)
    with pytest.raises(api.DsrgError):     # potts and compat together
        eng.crf_forward_train_wide_feat_dev(u, f, p, q, potts=torch.ones(2, device="cuda"),
                                            compat=torch.zeros((2, 40, 40), device="cuda"))
    assert eng.take_launch_count() == 0
    eng.close()


@pytest.mark.parametrize("what", ["theta", "features"])
def test_small_label_counts_are_dense_crf(torch_cuda, what):
    """At 32 labels or fewer dense_crf_wide passes theta and features to dense_crf: the same results up to the fused
    splat's float atomics."""
    torch = torch_cuda
    images = helpers.fused_images("smooth")
    B, H, W = images.shape[:3]
    unary, G = inputs(B, H, W, 21, 6)
    p = grad_params(1.0, 3)
    im = torch.from_numpy(images).cuda()
    feats = _nchw(torch, np.stack([features_of("guide", images[b], p, b) for b in range(B)]))
    res = []
    for fn in (nn.dense_crf, nn.dense_crf_wide):
        u = _nchw(torch, unary).requires_grad_(True)
        if what == "theta":
            th = torch.tensor([p.theta_gamma_x, p.theta_gamma_y], dtype=torch.float64, requires_grad=True)
            (fn(u, im, maxiter=3, theta_sp=th) * _nchw(torch, G)).sum().backward()
            res.append((u.grad, th.grad))
        else:
            f = feats.clone().requires_grad_(True)
            (fn(u, None, maxiter=3, features_bi=f) * _nchw(torch, G)).sum().backward()
            res.append((u.grad, f.grad))
    for a, b in zip(*res):
        assert torch.allclose(a, b, rtol=1e-5, atol=1e-6 * float(a.abs().max())), float((a - b).abs().max())
