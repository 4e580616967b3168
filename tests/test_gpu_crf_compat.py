"""The device's compatibility-matrix CRF (dsrg_crf_forward_train_compat_dev + dsrg_crf_backward_compat_dev,
nn.dense_crf(compat_bi=..., compat_sp=...)) against the float64 restatement of oracle/crf_compat_oracle.py, each case
under its own bar (tests/crf_compat_cases.py: BAR_K times the float32 models' noise of that case), and against the
reference's MatrixCompatibility through the frozen tests/golden/crf_compat_grad_ref.npz.

Cases: every tile path of the fused kernels (shared-memory tiles, direct tiles of either lattice, hybrid tiles, each
asserted reached), tail1 (21 labels in 24 lanes, 1 in 4) and phantom lanes (2 and 6 labels), 32 labels, non-square
images, B = 2 with distinct images, T = 0..10, mu = 0, -w I, symmetric, diagonal, w (1 - I) and non-symmetric; -w I
against the device's Potts path; graphs on and off, a cached graph replayed after mu changed in
place, another pass between forward and backward; nn.dense_crf in a CUDA graph; refusals before any launch."""
import ctypes as C
import os

import numpy as np
import pytest

import helpers
from crf_compat_cases import COMPAT_ITERS, COMPAT_M, GOLDEN, GOLDEN_CASES, CompatTruth, compat_mats, golden_inputs
from crf_grad_cases import GradTruth, grad_params, upstream
from dsrg_b200 import _lib, api
from oracle import meanfield64

pytestmark = pytest.mark.gpu


def _nchw(torch, a):
    return torch.from_numpy(np.ascontiguousarray(np.transpose(a, (0, 3, 1, 2)))).cuda()


def _nhwc(t):
    return np.transpose(t.cpu().numpy(), (0, 2, 3, 1))


def _compat(torch, mus):
    return torch.from_numpy(np.stack(mus)).cuda()


def device_compat(torch, eng, image, unary, G, p, compat, stream=None):
    """-> (Q_T (B, H, W, M), dL/dunary (B, H, W, M), dL/dmu (B, 2, M, M)) from the two entry points; compat a device
    (2, M, M) tensor."""
    B, M = unary.shape[0], unary.shape[-1]
    u, g, im = _nchw(torch, unary), _nchw(torch, G), torch.from_numpy(image).cuda()
    q_hist = torch.empty((p.n_iters + 1,) + tuple(u.shape), device="cuda")
    gu, gm = torch.empty_like(u), torch.empty((B, 2, M, M), device="cuda")
    eng.crf_forward_train_compat_dev(u, im, p, compat, q_hist, stream=stream)
    eng.crf_backward_compat_dev(q_hist, im, p, compat, g, gu, grad_compat=gm, stream=stream)
    torch.cuda.synchronize()
    return _nhwc(q_hist[p.n_iters]), _nhwc(gu), gm.cpu().numpy()


def inputs(images, M, seed):
    B, H, W = images.shape[:3]
    unary = helpers.log_unary(B, H, W, M, seed, scale=1.0)
    G = np.stack([upstream(H, W, M, seed + b) for b in range(B)])
    return unary, G


def truths(images, unary, G, p, mus, compare=None):
    B = images.shape[0]
    return {b: CompatTruth(meanfield64.Problem(images[b], p), unary[b], G[b], p.n_iters, mus)
            for b in (range(B) if compare is None else compare)}


def check_batch(torch, images, M, p, mus, seed, compare=None, eng=None):
    B, H, W = images.shape[:3]
    unary, G = inputs(images, M, seed)
    eng = eng or api.Engine(B, H, W, M)
    q, gu, gm = device_compat(torch, eng, images, unary, G, p, _compat(torch, mus))
    for b, t in truths(images, unary, G, p, mus, compare).items():
        t.check(q[b], gu[b], gm[b], "image %d:" % b)
    return eng


def sm_count(torch):
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


PATH_CASES = [(path, M, T) for path in sorted(helpers.MF64_PATH_CONFIG) for M in (6, 21, 32) for T in (2, 10)]


@pytest.mark.parametrize("path,M,T", PATH_CASES)
def test_compat_on_every_tile_path(torch_cuda, path, M, T):
    img, sf = helpers.MF64_PATH_CONFIG[path]
    images = helpers.fused_images(img)
    pred = helpers.predict_tile_paths(images, sf, sm_count(torch_cuda))
    want = {"smem": ("bi", "smem"), "bi_direct": ("bi", "direct"), "sp_direct": ("sp", "direct")}[path]
    assert (np.asarray(pred[want[0]]) == want[1]).any(), "the case does not reach %s" % path
    check_batch(torch_cuda, images, M, grad_params(sf, T), compat_mats("nonsym", M, M + T), 100 + M + T)


@pytest.mark.parametrize("M", COMPAT_M)
def test_compat_at_every_label_count(torch_cuda, M):
    """tail1 at 1 and 21 labels, phantom lanes at 2 and 6, none at 24 and 32."""
    check_batch(torch_cuda, helpers.fused_images("smooth"), M, grad_params(1.0, 3), compat_mats("nonsym", M, M), 3 + M)


@pytest.mark.parametrize("T", COMPAT_ITERS)
def test_compat_at_every_iteration_count(torch_cuda, T):
    check_batch(torch_cuda, helpers.fused_images("noise"), 21, grad_params(1.0, T), compat_mats("nonsym", 21, T), 7)


@pytest.mark.parametrize("kind", ["zero", "potts", "sym", "diag", "classic", "nonsym"])
def test_compat_matrix_kinds(torch_cuda, kind):
    check_batch(torch_cuda, helpers.fused_images("smooth"), 6, grad_params(1.0, 3), compat_mats(kind, 6, 5), 9)


def test_compat_on_hybrid_tiles(torch_cuda):
    images = helpers.hybrid_images()
    eng = check_batch(torch_cuda, images, 21, grad_params(1.0, 2), compat_mats("nonsym", 21, 1), 13, compare=[0])
    assert eng.hybrid_tiles > 0


@pytest.mark.parametrize("name", sorted(GOLDEN_CASES))
def test_compat_pinned_to_the_reference(torch_cuda, name):
    """The device and the reference's own float32 MatrixCompatibility (frozen) lie within the bar of the truth."""
    image, unary, G, p, mus = golden_inputs(name)
    H, W, M = unary.shape
    q, gu, gm = device_compat(torch_cuda, api.Engine(1, H, W, M), image[None], unary[None], G[None], p,
                              _compat(torch_cuda, mus))
    truth = CompatTruth(meanfield64.Problem(image, p), unary, G, p.n_iters, mus)
    with np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", GOLDEN)) as z:
        truth.check(z[name + "/q"], z[name + "/grad_unary"], None, "reference:")
    truth.check(q[0], gu[0], gm[0], "device:")


def test_potts_matrices_agree_with_the_potts_path(torch_cuda):
    """mu = -w I against dsrg_crf_backward_dev on the same inputs: dL/dU within the bars, -trace(dL/dmu_k) = dL/dw_k."""
    torch = torch_cuda
    images = helpers.fused_images("noise")
    B, H, W = images.shape[:3]
    M, T = 6, 3
    p = grad_params(1.0, T, w1=4.0, w2=2.0)
    mus = compat_mats("potts", M, 0, p.w1, p.w2)
    unary, G = inputs(images, M, 31)
    eng = api.Engine(B, H, W, M)
    q, gu, gm = device_compat(torch, eng, images, unary, G, grad_params(1.0, T), _compat(torch, mus))
    u, g, im = _nchw(torch, unary), _nchw(torch, G), torch.from_numpy(images).cuda()
    q_hist = torch.empty((T + 1,) + tuple(u.shape), device="cuda")
    gu_p, gw_p = torch.empty_like(u), torch.empty((B, 2), device="cuda")
    eng.crf_forward_train_dev(u, im, p, q_hist)
    eng.crf_backward_dev(q_hist, im, p, g, gu_p, grad_potts=gw_p)
    torch.cuda.synchronize()
    gu_p, gw_p, q_p = _nhwc(gu_p), gw_p.cpu().numpy(), _nhwc(q_hist[T])
    for b, t in truths(images, unary, G, p, mus).items():
        gt = GradTruth(meanfield64.Problem(images[b], p), unary[b], G[b], T)
        t.check(q[b], gu[b], gm[b], "compat image %d:" % b)
        assert np.abs(q[b] - q_p[b]).max() <= 2 * t.bar_q
        assert np.abs(gu[b] - gu_p[b]).max() <= t.bar_u + gt.bar_u
        for i in (0, 1):
            bar = np.trace(t.bar_mu[i]) + gt.bar_w[i]
            assert abs(-np.trace(gm[b, i]) - gw_p[b, i]) <= bar, (b, i, -np.trace(gm[b, i]), gw_p[b, i], bar)


def test_graphs_in_place_update_and_another_pass_in_between(torch_cuda):
    torch = torch_cuda
    images = helpers.fused_images("smooth")
    B, H, W = images.shape[:3]
    M, T = 24, 3
    p = grad_params(1.0, T)
    unary, G = inputs(images, M, 41)
    mus_a, mus_b = compat_mats("nonsym", M, 1), compat_mats("sym", M, 2)
    ta, tb = truths(images, unary, G, p, mus_a), truths(images, unary, G, p, mus_b)
    eng = api.Engine(B, H, W, M)
    c = _compat(torch, mus_a)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        r0 = eng.graph_replays
        for _ in range(3):   # eager, captured, replayed
            q, gu, gm = device_compat(torch, eng, images, unary, G, p, c, stream=s.cuda_stream)
            for b in range(B):
                ta[b].check(q[b], gu[b], gm[b], "graphs on:")
        r1 = eng.graph_replays
        assert r1 > r0
        c.copy_(_compat(torch, mus_b))   # the same address, new values: the cached graphs replay and read them
        q, gu, gm = device_compat(torch, eng, images, unary, G, p, c, stream=s.cuda_stream)
        assert eng.graph_replays > r1
        for b in range(B):
            tb[b].check(q[b], gu[b], gm[b], "after an in-place update:")
        # another pass between the forward and the backward: other images, other sigmas
        u, g, im = _nchw(torch, unary), _nchw(torch, G), torch.from_numpy(images).cuda()
        q_hist = torch.empty((T + 1,) + tuple(u.shape), device="cuda")
        gu_t, gm_t = torch.empty_like(u), torch.empty((B, 2, M, M), device="cuda")
        eng.crf_forward_train_compat_dev(u, im, p, c, q_hist, stream=s.cuda_stream)
        out = torch.empty_like(u)
        eng.crf_dev(u, torch.from_numpy(np.ascontiguousarray(images[::-1])).cuda(), api.crf_params(12.0), out,
                    unary_layout=api.LAYOUT_NCHW, out_layout=api.LAYOUT_NCHW, stream=s.cuda_stream)
        eng.crf_backward_compat_dev(q_hist, im, p, c, g, gu_t, grad_compat=gm_t, stream=s.cuda_stream)
        torch.cuda.synchronize()
        for b in range(B):
            tb[b].check(_nhwc(q_hist[T])[b], _nhwc(gu_t)[b], gm_t.cpu().numpy()[b], "pass in between:")
    with pytest.raises(api.DsrgError) as e:
        eng.crf_last_marginals_host(B)
    assert e.value.code == _lib.E_STATE
    eng.set_graphs(False)
    q, gu, gm = device_compat(torch, eng, images, unary, G, p, c)
    for b in range(B):
        tb[b].check(q[b], gu[b], gm[b], "graphs off:")


def test_dense_crf_compat_in_a_cuda_graph(torch_cuda):
    """nn.dense_crf(compat_bi=mu, w2=w) captured in a torch.cuda.CUDAGraph: the gradients to the unary, to mu and to
    w (through the -w I built for the spatial term) equal the eager ones and the truth's batch sums."""
    torch = torch_cuda
    from dsrg_b200 import nn
    images = helpers.fused_images("smooth")
    B, H, W = images.shape[:3]
    M, T = 21, 5
    unary, G = inputs(images, M, 51)
    im = torch.from_numpy(images).cuda()
    u0, g0 = _nchw(torch, unary), _nchw(torch, G)
    mu_bi = compat_mats("nonsym", M, 3)[0]
    w2v = 3.0

    def step(u, mu, w2):
        q = nn.dense_crf(u, im, scale_factor=1.0, maxiter=T, compat_bi=mu, w2=w2)
        (q * g0).sum().backward()
        return q

    u = u0.clone().requires_grad_(True)
    mu = torch.from_numpy(mu_bi).cuda().requires_grad_(True)
    w2 = torch.tensor(w2v, device="cuda", requires_grad=True)
    q_eager = step(u, mu, w2).detach().clone()
    eager = (u.grad.clone(), mu.grad.clone(), w2.grad.clone())
    p = grad_params(1.0, T)
    mus = (mu_bi, np.float32(-w2v) * np.eye(M, dtype=np.float32))
    tr = truths(images, unary, G, p, mus)
    for b in range(B):
        tr[b].check(_nhwc(q_eager)[b], _nhwc(eager[0])[b], None, "eager image %d:" % b)
    want_mu = sum(tr[b].gmu[0] for b in range(B))
    bar_mu = sum(tr[b].bar_mu[0] for b in range(B))
    assert (np.abs(eager[1].cpu().numpy() - want_mu) <= bar_mu).all()
    want_w2 = -sum(np.trace(tr[b].gmu[1]) for b in range(B))
    bar_w2 = sum(np.trace(tr[b].bar_mu[1]) for b in range(B))
    assert abs(float(eager[2]) - want_w2) <= bar_w2, (float(eager[2]), want_w2, bar_w2)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):   # warm-up on the side stream, as torch.cuda.graphs asks
        for t in (u, mu, w2):
            t.grad = None
        step(u, mu, w2)
    torch.cuda.current_stream().wait_stream(s)
    for t in (u, mu, w2):
        t.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        q_static = step(u, mu, w2)
    for t in (u, mu, w2):
        t.grad.zero_()
    graph.replay()
    torch.cuda.synchronize()
    np.testing.assert_allclose(q_static.detach().cpu().numpy(), q_eager.cpu().numpy(), atol=1e-5)
    assert float((u.grad - eager[0]).abs().max()) <= 2 * max(tr[b].bar_u for b in range(B))
    assert (np.abs(mu.grad.cpu().numpy() - eager[1].cpu().numpy()) <= 2 * bar_mu).all()
    assert abs(float(w2.grad) - float(eager[2])) <= 2 * bar_w2


def test_refusals_before_any_launch(torch_cuda):
    torch = torch_cuda
    from dsrg_b200 import nn
    L = _lib.lib()
    ptr = api._dptr
    # 33 labels
    B, H, W, M = 1, 9, 11, 33
    eng = api.Engine(B, H, W, M)
    u = torch.zeros((B, M, H, W), device="cuda")
    im = torch.zeros((B, H, W, 3), dtype=torch.uint8, device="cuda")
    q_hist = torch.empty((3, B, M, H, W), device="cuda")
    c = torch.zeros((2, M, M), device="cuda")
    p = grad_params(1.0, 2)
    eng.take_launch_count()
    with pytest.raises(api.DsrgError) as e:
        eng.crf_forward_train_compat_dev(u, im, p, c, q_hist)
    assert e.value.code == _lib.E_INVALID and "32 labels" in str(e.value)
    with pytest.raises(api.DsrgError) as e:
        eng.crf_backward_compat_dev(q_hist, im, p, c, u, torch.empty_like(u))
    assert e.value.code == _lib.E_INVALID
    assert eng.take_launch_count() == 0
    with pytest.raises(ValueError):
        nn.dense_crf(u, im, compat_bi=torch.zeros((M, M), device="cuda"))
    # out-of-range batches and a missing matrix
    B, M = 2, 6
    eng = api.Engine(B, H, W, M)
    u = torch.zeros((B, M, H, W), device="cuda")
    im = torch.zeros((B, H, W, 3), dtype=torch.uint8, device="cuda")
    q_hist = torch.empty((3, B, M, H, W), device="cuda")
    c = torch.zeros((2, M, M), device="cuda")
    eng.take_launch_count()
    for bad in (0, B + 1):
        for rc in (L.dsrg_crf_forward_train_compat_dev(eng.h, ptr(u), bad, ptr(im), C.byref(p), ptr(c), ptr(q_hist),
                                                       None),
                   L.dsrg_crf_backward_compat_dev(eng.h, ptr(q_hist), bad, ptr(im), C.byref(p), ptr(c), ptr(u),
                                                  ptr(u), None, None)):
            assert rc == _lib.E_INVALID
            assert "batch %d outside [1, %d]" % (bad, B) in L.dsrg_last_error().decode()
    assert L.dsrg_crf_forward_train_compat_dev(eng.h, ptr(u), B, ptr(im), C.byref(p), None, ptr(q_hist),
                                               None) == _lib.E_INVALID
    assert eng.take_launch_count() == 0
    # the Python checks: shapes, dtype, device, and a matrix together with its weight
    good = torch.zeros((M, M), device="cuda")
    for bad in (torch.zeros((M, M + 1), device="cuda"), torch.zeros((M,), device="cuda"),
                torch.zeros((M, M), dtype=torch.int32, device="cuda"), torch.zeros((M, M)), np.zeros((M, M))):
        with pytest.raises(ValueError):
            nn.dense_crf(u, im, compat_bi=bad)
        with pytest.raises(ValueError):
            nn.dense_crf(u, im, compat_sp=bad)
    with pytest.raises(ValueError):
        nn.dense_crf(u, im, compat_bi=good, w1=torch.tensor(1.0, device="cuda"))
    with pytest.raises(ValueError):
        nn.dense_crf(u, im, compat_sp=good, w2=torch.tensor(1.0, device="cuda"))
    assert eng.take_launch_count() == 0
