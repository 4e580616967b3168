"""The device's kernel-bandwidth gradient (dsrg_crf_backward_theta_dev, dsrg_crf_backward_compat_theta_dev,
nn.dense_crf(theta_bi=..., theta_sp=...)) against the float64 exact derivative of oracle/crf_kgrad_oracle.py.

Bar: per case and per component, tests/crf_kgrad_cases.KgradTruth's: BAR_K times the float32 models' error, with a
floor from the magnitude of the terms; test_crf_kgrad_cpu.py shows every mutant outside these bars on every case.

Cases: every tile path of the fused kernels for the backward's g_t store, small shapes with phantom lanes, B = 2 with
distinct images, M in {1, 2, 6, 21, 24, 32}, T in {0, 1, 2, 3, 10}, anisotropic and per-channel sigmas, Potts with
host and device weights, and a non-symmetric mu; grad_unary and the Potts / compatibility gradients of the new entry
points against the existing ones; graphs on and off and another pass in between; the refusals."""
import numpy as np
import pytest

import helpers
from crf_compat_cases import compat_mats
from crf_grad_cases import grad_params
from crf_kgrad_cases import (ITERS, LABELS, PATH_MT, SET_MU, SET_NAMES, KgradTruth, inputs, label_case,
                             label_case_runs, path_case, set_case)
from dsrg_b200 import _lib, api

pytestmark = pytest.mark.gpu


def _nchw(torch, a):
    return torch.from_numpy(np.ascontiguousarray(np.transpose(a, (0, 3, 1, 2)))).cuda()


def device_theta(torch, eng, images, unary, G, p, mus=None, potts=None):
    """-> (grad_theta (B, 7), grad_unary (B, M, H, W), grad of the weights / matrices) from the new entry points."""
    B, M = unary.shape[0], unary.shape[-1]
    u, g, im = _nchw(torch, unary), _nchw(torch, G), torch.from_numpy(images).cuda()
    q_hist = torch.empty((p.n_iters + 1,) + tuple(u.shape), device="cuda")
    gu, gt = torch.empty_like(u), torch.full((B, 7), float("nan"), device="cuda")
    if mus is not None:
        compat = torch.from_numpy(np.stack(mus).astype(np.float32)).cuda()
        gw = torch.empty((B, 2, M, M), device="cuda")
        eng.crf_forward_train_compat_dev(u, im, p, compat, q_hist)
        eng.crf_backward_compat_theta_dev(q_hist, im, p, compat, g, gu, gt, grad_compat=gw)
    else:
        gw = torch.empty((B, 2), device="cuda")
        eng.crf_forward_train_dev(u, im, p, q_hist, potts=potts)
        eng.crf_backward_theta_dev(q_hist, im, p, g, gu, gt, grad_potts=gw, potts=potts)
    torch.cuda.synchronize()
    return gt.cpu().numpy(), gu.cpu().numpy(), gw.cpu().numpy()


def check_theta(images, unary, G, p, got, mus=None, compare=None):
    for b in (range(images.shape[0]) if compare is None else compare):
        KgradTruth(images[b], p, unary[b], G[b], mus).check(got[b], "image %d:" % b)


def run_case(torch, case, potts=None):
    images, p, unary, G, mus, compare = case
    B, H, W = images.shape[:3]
    eng = api.Engine(B, H, W, unary.shape[-1])
    got = device_theta(torch, eng, images, unary, G, p, mus, potts)
    check_theta(images, unary, G, p, got[0], mus, compare)
    eng.close()
    return got


def sm_count(torch):
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


@pytest.mark.parametrize("path,M,T", [(path, M, T) for path in sorted(helpers.MF64_PATH_CONFIG) for M, T in PATH_MT])
def test_theta_on_every_tile_path(torch_cuda, path, M, T):
    img, sf = helpers.MF64_PATH_CONFIG[path]
    images = helpers.fused_images(img)
    pred = helpers.predict_tile_paths(images, sf, sm_count(torch_cuda))
    want = {"smem": ("bi", "smem"), "bi_direct": ("bi", "direct"), "sp_direct": ("sp", "direct")}[path]
    assert (np.asarray(pred[want[0]]) == want[1]).any(), "the case does not reach %s" % path
    run_case(torch_cuda, path_case(path, M, T))


@pytest.mark.parametrize("M", LABELS)
@pytest.mark.parametrize("T", ITERS)
def test_theta_labels_and_iterations(torch_cuda, M, T):
    if not label_case_runs(M, T):
        pytest.skip("ten iterations at two label counts")
    got = run_case(torch_cuda, label_case(M, T))
    if T == 0 or M == 1:
        assert not np.any(got[0]), got[0]


@pytest.mark.parametrize("name", SET_NAMES)
@pytest.mark.parametrize("mu", SET_MU)
def test_theta_at_parameter_sets(torch_cuda, name, mu):
    case = set_case(name, mu)
    p = case[1]
    potts = torch_cuda.tensor([p.w1, p.w2], device="cuda") if mu == "potts_dev" else None
    run_case(torch_cuda, case, potts=potts)


@pytest.mark.parametrize("mu", [None, "nonsym"])
def test_other_gradients_match_the_existing_backward(torch_cuda, mu):
    torch = torch_cuda
    images = helpers.fused_images("noise")
    B, H, W = images.shape[:3]
    M, p = 21, grad_params(1.0, 3)
    unary, G = inputs(images, M, 500)
    mus = compat_mats(mu, M, 5) if mu else None
    eng = api.Engine(B, H, W, M)
    _, gu_t, gw_t = device_theta(torch, eng, images, unary, G, p, mus)
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
    # the same kernels; only the order of the float atomics in the splats differs between two runs
    np.testing.assert_allclose(gu_t, gu.cpu().numpy(), rtol=0, atol=1e-4 * float(np.abs(gu_t).max()))
    np.testing.assert_allclose(gw_t, gw.cpu().numpy(), rtol=1e-3, atol=1e-4 * float(np.abs(gw_t).max()))
    eng.close()


@pytest.mark.parametrize("graphs", [0, 1])
def test_graphs_and_an_intervening_pass(torch_cuda, graphs):
    torch = torch_cuda
    images = helpers.fused_images("smooth")
    B, H, W = images.shape[:3]
    M, p = 6, grad_params(1.0, 2)
    unary, G = inputs(images, M, 600)
    eng = api.Engine(B, H, W, M)
    _lib.lib().dsrg_engine_set_graphs(eng.h, graphs)
    first = device_theta(torch, eng, images, unary, G, p)[0]
    # another pass with other sigmas on the same engine, then the same backward again (a replayed graph when on)
    out = torch.empty((B, M, H, W), device="cuda")
    eng.crf_dev(_nchw(torch, unary), torch.from_numpy(images).cuda(), api.crf_params(12.0), out,
                unary_layout=api.LAYOUT_NCHW, out_layout=api.LAYOUT_NCHW)
    again = device_theta(torch, eng, images, unary, G, p)[0]
    check_theta(images, unary, G, p, first)
    check_theta(images, unary, G, p, again)
    eng.close()


def test_refusals(torch_cuda):
    torch = torch_cuda
    H, W, M = 9, 11, 3
    eng = api.Engine(2, H, W, M)
    p = grad_params(1.0, 2)
    u = torch.zeros((2, M, H, W), device="cuda")
    im = torch.zeros((2, H, W, 3), dtype=torch.uint8, device="cuda")
    q = torch.zeros((3, 2, M, H, W), device="cuda")
    gt = torch.zeros((2, 7), device="cuda")
    with pytest.raises(api.DsrgError):     # grad_theta is required
        eng.crf_backward_theta_dev(q, im, p, u, torch.empty_like(u), None)
    compat = torch.zeros((2, M, M), device="cuda")
    with pytest.raises(api.DsrgError):
        eng.crf_backward_compat_theta_dev(q, im, p, compat, u, torch.empty_like(u), None)
    big = torch.zeros((3, M, H, W), device="cuda")
    with pytest.raises(api.DsrgError):     # batch above the engine's
        eng.crf_backward_theta_dev(torch.zeros((3, 3, M, H, W), device="cuda"), im, p, big, torch.empty_like(big),
                                   torch.zeros((3, 7), device="cuda"))
    eng.close()
    eng33 = api.Engine(1, H, W, 33)
    u33 = torch.zeros((1, 33, H, W), device="cuda")
    with pytest.raises(api.DsrgError):
        eng33.crf_backward_theta_dev(torch.zeros((3, 1, 33, H, W), device="cuda"), im[:1], p, u33,
                                     torch.empty_like(u33), gt[:1])
    eng33.close()


@pytest.mark.parametrize("where", ["cpu", "cuda"])
@pytest.mark.parametrize("mu", [None, "nonsym"])
def test_dense_crf_learns_theta(torch_cuda, where, mu):
    torch = torch_cuda
    from dsrg_b200 import nn
    images = helpers.fused_images("noise")
    B, H, W = images.shape[:3]
    M, T = 6, 3
    unary, G = inputs(images, M, 700)
    p = api.crf_params(1.0, 13, T)
    th_bi = torch.tensor([p.theta_alpha_x, p.theta_alpha_y, p.theta_beta_r, p.theta_beta_g, p.theta_beta_b],
                         dtype=torch.float64, device=where, requires_grad=True)
    th_sp = torch.tensor([p.theta_gamma_x, p.theta_gamma_y], dtype=torch.float64, device=where, requires_grad=True)
    kw = {}
    mus = None
    if mu:
        mus = compat_mats(mu, M, 3)
        kw = dict(compat_bi=torch.from_numpy(mus[0].astype(np.float32)).cuda(),
                  compat_sp=torch.from_numpy(mus[1].astype(np.float32)).cuda())
    u = _nchw(torch, unary)
    q = nn.dense_crf(u, torch.from_numpy(images).cuda(), 1.0, 13, T, theta_bi=th_bi, theta_sp=th_sp, **kw)
    (q * _nchw(torch, G)).sum().backward()
    assert th_bi.grad.device == th_bi.device and th_bi.grad.dtype == torch.float64
    got = np.concatenate([th_bi.grad.cpu().numpy(), th_sp.grad.cpu().numpy()])
    want, bar = np.zeros(7), np.zeros(7)
    for b in range(B):
        t = KgradTruth(images[b], p, unary[b], G[b], mus)
        want += t.want
        bar += t.bar
    assert np.all(np.abs(got - want) <= bar), (got, want, bar)


@pytest.mark.parametrize("where", ["cpu", "cuda"])
def test_dense_crf_refuses_theta_in_capture(torch_cuda, where):
    torch = torch_cuda
    from dsrg_b200 import nn
    u = torch.zeros((1, 3, 9, 11), device="cuda")
    im = torch.zeros((1, 9, 11, 3), dtype=torch.uint8, device="cuda")
    th = torch.ones(2, device=where)
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        g.capture_begin()
        try:
            with pytest.raises(ValueError, match="capture"):
                nn.dense_crf(u, im, theta_sp=th)
        finally:
            g.capture_end()
