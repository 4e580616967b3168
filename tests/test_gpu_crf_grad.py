"""The device's CRF gradient (dsrg_crf_forward_train_dev + dsrg_crf_backward_dev, nn.dense_crf) against the float64
backward of oracle/crf_grad_oracle.py, each case under its own bar (tests/crf_grad_cases.py: BAR_K times the float32
models' noise of that case), and against the reference's own gradient through the frozen tests/golden/crf_grad_ref.npz.

Cases: every tile path of the fused kernels (shared-memory tiles, direct tiles of either lattice, hybrid tiles) with
tail1 (21 labels in 24 lanes) and not, non-square images, B = 2 with distinct images, T = 0..10, each Potts weight
zeroed; the marginals the forward keeps; device-resident Potts weights; graphs on and off; another pass between the
forward and the backward; nn.dense_crf inside a CUDA graph; 33 labels refused; the retained-marginals state."""
import ctypes as C
import os

import numpy as np
import pytest

import helpers
from crf_grad_cases import GOLDEN, GOLDEN_CASES, GradTruth, golden_inputs, grad_params, upstream
from dsrg_b200 import _lib, api
from oracle import meanfield64

pytestmark = pytest.mark.gpu


def _nchw(torch, a):
    return torch.from_numpy(np.ascontiguousarray(np.transpose(a, (0, 3, 1, 2)))).cuda()


def _nhwc(t):
    return np.transpose(t.cpu().numpy(), (0, 2, 3, 1))


def device_grad(torch, eng, image, unary, G, p, potts=None, stream=None):
    """-> (q_hist (T+1, B, H, W, M), dL/dunary (B, H, W, M), dL/dw (B, 2)) from the two entry points."""
    B = unary.shape[0]
    u, g, im = _nchw(torch, unary), _nchw(torch, G), torch.from_numpy(image).cuda()
    q_hist = torch.empty((p.n_iters + 1,) + tuple(u.shape), device="cuda")
    gu, gw = torch.empty_like(u), torch.empty((B, 2), device="cuda")
    eng.crf_forward_train_dev(u, im, p, q_hist, potts=potts, stream=stream)
    eng.crf_backward_dev(q_hist, im, p, g, gu, grad_potts=gw, potts=potts, stream=stream)
    torch.cuda.synchronize()
    return np.transpose(q_hist.cpu().numpy(), (0, 1, 3, 4, 2)), _nhwc(gu), gw.cpu().numpy()


def inputs(images, M, seed):
    B, H, W = images.shape[:3]
    unary = helpers.log_unary(B, H, W, M, seed, scale=1.0)
    G = np.stack([upstream(H, W, M, seed + b) for b in range(B)])
    return unary, G


def check_batch(torch, images, M, p, seed, compare=None, eng=None, potts=None):
    B, H, W = images.shape[:3]
    unary, G = inputs(images, M, seed)
    eng = eng or api.Engine(B, H, W, M)
    _, gu, gw = device_grad(torch, eng, images, unary, G, p, potts=potts)
    for b in (range(B) if compare is None else compare):
        truth = GradTruth(meanfield64.Problem(images[b], p), unary[b], G[b], p.n_iters)
        truth.check(gu[b], gw[b], "image %d:" % b)
    return eng


PATH_CASES = [(path, M, T) for path in sorted(helpers.MF64_PATH_CONFIG) for M in (6, 21, 32) for T in (2, 10)]


@pytest.mark.parametrize("path,M,T", PATH_CASES)
def test_gradient_on_every_tile_path(torch_cuda, path, M, T):
    img, sf = helpers.MF64_PATH_CONFIG[path]
    check_batch(torch_cuda, helpers.fused_images(img), M, grad_params(sf, T), 100 + M + T)


@pytest.mark.parametrize("T", [0, 1, 3])
def test_gradient_at_few_iterations(torch_cuda, T):
    check_batch(torch_cuda, helpers.fused_images("smooth"), 21, grad_params(1.0, T), 7)


@pytest.mark.parametrize("zero", ["w1", "w2"])
def test_gradient_with_one_potts_weight_zeroed(torch_cuda, zero):
    check_batch(torch_cuda, helpers.fused_images("noise"), 6, grad_params(1.0, 3, zero), 9)


def test_gradient_on_hybrid_tiles(torch_cuda):
    images = helpers.hybrid_images()
    eng = check_batch(torch_cuda, images, 21, grad_params(1.0, 2), 13, compare=[0])
    assert eng.hybrid_tiles > 0   # the backward's own lattice build had hybrid tiles


@pytest.mark.parametrize("name", sorted(GOLDEN_CASES))
def test_gradient_pinned_to_the_reference(torch_cuda, name):
    """The device and the reference's own float32 gradient (frozen) both lie within the bar of the float64 truth."""
    image, unary, G, p = golden_inputs(name)
    H, W, M = unary.shape
    eng = api.Engine(1, H, W, M)
    _, gu, gw = device_grad(torch_cuda, eng, image[None], unary[None], G[None], p)
    truth = GradTruth(meanfield64.Problem(image, p), unary, G, p.n_iters)
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", GOLDEN))
    truth.check(z[name + "/grad_unary"], z[name + "/grad_potts"], "reference:")
    truth.check(gu[0], gw[0], "device:")


def test_history_holds_the_forward_marginals(torch_cuda):
    """q_hist[T] against dsrg_crf_batch_dev's marginals and both against the float64 forward, within its bar."""
    torch = torch_cuda
    images = helpers.fused_images("smooth")
    B, H, W = images.shape[:3]
    M, T = 21, 10
    p = grad_params(1.0, T)
    unary, G = inputs(images, M, 21)
    eng = api.Engine(B, H, W, M)
    q_hist, _, _ = device_grad(torch, eng, images, unary, G, p)
    with pytest.raises(api.DsrgError) as e:   # the marginals are the caller's q_hist, not the engine's
        eng.crf_last_marginals_host(B)
    assert e.value.code == _lib.E_STATE
    out = torch.empty((B, M, H, W), device="cuda")
    eng.crf_dev(_nchw(torch, unary), torch.from_numpy(images).cuda(), p, out, unary_layout=api.LAYOUT_NCHW,
                out_layout=api.LAYOUT_NCHW)
    q = _nhwc(out)
    for b in range(B):
        P = meanfield64.Problem(images[b], p)
        q64, bar, _, _ = helpers.mf64_truth_and_bar(P, unary[b], iters=(1, T))
        for n in (1, T):
            assert np.abs(q_hist[n, b] - q64[n]).max() <= bar[n], (b, n)
        assert np.abs(q[b] - q64[T]).max() <= bar[T]
        np.testing.assert_allclose(q_hist[0, b], P.run(unary[b], 0)[0], atol=1e-6)


def test_device_potts_weights_equal_params(torch_cuda):
    torch = torch_cuda
    images = helpers.fused_images("noise")
    B, H, W = images.shape[:3]
    p = grad_params(1.0, 3, w1=4.0, w2=2.0)
    unary, G = inputs(images, 6, 31)
    eng = api.Engine(B, H, W, 6)
    base = grad_params(1.0, 3)   # CRF()'s 10 and 3: the device weights must win over these
    potts = torch.tensor([4.0, 2.0], device="cuda")
    q1, gu1, gw1 = device_grad(torch, eng, images, unary, G, base, potts=potts)
    q2, gu2, gw2 = device_grad(torch, eng, images, unary, G, p)
    for b in range(B):
        truth = GradTruth(meanfield64.Problem(images[b], p), unary[b], G[b], 3)
        truth.check(gu1[b], gw1[b], "potts_dev:")
        truth.check(gu2[b], gw2[b], "params:")


def test_graphs_on_and_off_and_another_pass_in_between(torch_cuda):
    torch = torch_cuda
    images = helpers.fused_images("smooth")
    B, H, W = images.shape[:3]
    M = 24
    p = grad_params(1.0, 3)
    unary, G = inputs(images, M, 41)
    truths = [GradTruth(meanfield64.Problem(images[b], p), unary[b], G[b], 3) for b in range(B)]
    eng = api.Engine(B, H, W, M)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        r0 = eng.graph_replays
        for _ in range(3):   # eager, captured, replayed
            _, gu, gw = device_grad(torch, eng, images, unary, G, p, stream=s.cuda_stream)
            for b in range(B):
                truths[b].check(gu[b], gw[b], "graphs on:")
        assert eng.graph_replays > r0
        # another pass between the forward and the backward: other images, other sigmas (the spatial lattice too)
        u, g, im = _nchw(torch, unary), _nchw(torch, G), torch.from_numpy(images).cuda()
        q_hist = torch.empty((4,) + tuple(u.shape), device="cuda")
        gu_t, gw_t = torch.empty_like(u), torch.empty((B, 2), device="cuda")
        eng.crf_forward_train_dev(u, im, p, q_hist, stream=s.cuda_stream)
        other = np.ascontiguousarray(images[::-1])
        out = torch.empty_like(u)
        eng.crf_dev(u, torch.from_numpy(other).cuda(), api.crf_params(12.0), out, unary_layout=api.LAYOUT_NCHW,
                    out_layout=api.LAYOUT_NCHW, stream=s.cuda_stream)
        eng.crf_backward_dev(q_hist, im, p, g, gu_t, grad_potts=gw_t, stream=s.cuda_stream)
        torch.cuda.synchronize()
        for b in range(B):
            truths[b].check(_nhwc(gu_t)[b], gw_t.cpu().numpy()[b], "pass in between:")
    eng.set_graphs(False)
    _, gu, gw = device_grad(torch, eng, images, unary, G, p)
    for b in range(B):
        truths[b].check(gu[b], gw[b], "graphs off:")


def test_dense_crf_autograd_in_a_cuda_graph(torch_cuda):
    torch = torch_cuda
    from dsrg_b200 import nn
    images = helpers.fused_images("smooth")
    B, H, W = images.shape[:3]
    M, T = 21, 5
    unary, G = inputs(images, M, 51)
    im = torch.from_numpy(images).cuda()
    u0, g0 = _nchw(torch, unary), _nchw(torch, G)

    def step(u, w1, w2):
        q = nn.dense_crf(u, im, scale_factor=1.0, maxiter=T, w1=w1, w2=w2)
        (q * g0).sum().backward()
        return q

    u = u0.clone().requires_grad_(True)
    w1 = torch.tensor(10.0, device="cuda", requires_grad=True)
    w2 = torch.tensor(3.0, device="cuda", requires_grad=True)
    q_eager = step(u, w1, w2).detach().clone()
    eager = (u.grad.clone(), w1.grad.clone(), w2.grad.clone())
    p = grad_params(1.0, T)
    for b in range(B):
        truth = GradTruth(meanfield64.Problem(images[b], p), unary[b], G[b], T)
        truth.check(_nhwc(eager[0])[b], None, "eager image %d:" % b)
    gw = np.array([float(eager[1]), float(eager[2])])
    truths = [GradTruth(meanfield64.Problem(images[b], p), unary[b], G[b], T) for b in range(B)]
    want = np.array([sum(t.gw[i] for t in truths) for i in (0, 1)])
    bars = np.array([sum(t.bar_w[i] for t in truths) for i in (0, 1)])
    assert (np.abs(gw - want) <= bars).all(), (gw, want, bars)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):   # warm-up on the side stream, as torch.cuda.graphs asks
        for t in (u, w1, w2):
            t.grad = None
        step(u, w1, w2)
    torch.cuda.current_stream().wait_stream(s)
    for t in (u, w1, w2):
        t.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        q_static = step(u, w1, w2)
    for t in (u, w1, w2):
        t.grad.zero_()
    graph.replay()
    torch.cuda.synchronize()
    np.testing.assert_allclose(q_static.detach().cpu().numpy(), q_eager.cpu().numpy(), atol=1e-5)
    for got, want_t, name in zip((u.grad, w1.grad, w2.grad), eager, ("unary", "w1", "w2")):
        tol = truths[0].bar_u if name == "unary" else bars[0 if name == "w1" else 1]
        assert float((got - want_t).abs().max()) <= 2 * tol, name


def test_more_than_32_labels_are_refused(torch_cuda):
    torch = torch_cuda
    from dsrg_b200 import nn
    B, H, W, M = 1, 9, 11, 33
    eng = api.Engine(B, H, W, M)
    u = torch.zeros((B, M, H, W), device="cuda")
    im = torch.zeros((B, H, W, 3), dtype=torch.uint8, device="cuda")
    q_hist = torch.empty((3, B, M, H, W), device="cuda")
    with pytest.raises(api.DsrgError) as e:
        eng.crf_forward_train_dev(u, im, grad_params(1.0, 2), q_hist)
    assert e.value.code == _lib.E_INVALID and "32 labels" in str(e.value)
    with pytest.raises(api.DsrgError) as e:
        eng.crf_backward_dev(q_hist, im, grad_params(1.0, 2), u, torch.empty_like(u))
    assert e.value.code == _lib.E_INVALID
    with pytest.raises(ValueError):
        nn.dense_crf(u, im)


def test_batch_range_is_refused_before_any_launch(torch_cuda):
    torch = torch_cuda
    B, H, W, M = 2, 9, 11, 6
    eng = api.Engine(B, H, W, M)
    L = _lib.lib()
    u = torch.zeros((B, M, H, W), device="cuda")
    im = torch.zeros((B, H, W, 3), dtype=torch.uint8, device="cuda")
    q_hist = torch.empty((3, B, M, H, W), device="cuda")
    p = grad_params(1.0, 2)
    ptr = api._dptr
    eng.take_launch_count()
    for bad in (0, B + 1):
        for rc in (L.dsrg_crf_forward_train_dev(eng.h, ptr(u), bad, ptr(im), C.byref(p), None, ptr(q_hist), None),
                   L.dsrg_crf_backward_dev(eng.h, ptr(q_hist), bad, ptr(im), C.byref(p), None, ptr(u), ptr(u),
                                           None, None)):
            assert rc == _lib.E_INVALID
            assert "batch %d outside [1, %d]" % (bad, B) in L.dsrg_last_error().decode()
    assert eng.take_launch_count() == 0
