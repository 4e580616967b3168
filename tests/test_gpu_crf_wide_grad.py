"""The dense CRF's gradient above 32 labels (dsrg_crf_forward_train_wide_dev + dsrg_crf_backward_wide_dev,
nn.dense_crf_wide) against the float64 restatements (oracle/crf_grad_oracle.py, oracle/crf_compat_oracle.py), each
case under its own bar (crf_grad_cases.GradTruth, crf_compat_cases.CompatTruth: BAR_K times the float32 models' noise
of that case).

Cases: M = 33, 36, 81, 128, 255 (phantom quad lanes and whole quads), T = 0, 1, 2, 10 at scale factors 1 and 12,
smooth, photo and noise images, host weights, device weights and non-symmetric matrices; slot-scaled batches (slot b
holds problem pi(b) with upstream s_b G); the shared spatial lattice rebuilt between calls, a batch below the engine's
and a re-shaped engine; an inference pass between forward and backward; the reference's own gradient at 81 labels
(frozen); COCO's training shape (batch 20 @ 41x41, sf 12, T = 10) through nn.dense_crf_wide, every slot; one 321x321
photo; a captured nn.dense_crf_wide step replayed with new unaries and weights; autocast; refusals before any launch."""
import os

import numpy as np
import pytest

import helpers
from crf_compat_cases import CompatTruth, compat_mats
from crf_grad_cases import GradTruth, grad_params, upstream
from crf_wide_grad_cases import GOLDEN, GOLDEN_CASES, WIDE_GRAD_M, golden_inputs
from dsrg_b200 import _lib, api, nn
from oracle import meanfield64

pytestmark = pytest.mark.gpu

SCALES = [1.0, -0.5, 2.0, -1.0]   # exact in float32: a slot's truth is s_b times its problem's


def _nchw(torch, a):
    return torch.from_numpy(np.ascontiguousarray(np.transpose(a, (0, 3, 1, 2)))).cuda()


def _nhwc(t):
    return np.transpose(t.detach().cpu().numpy(), (0, 2, 3, 1))


def device_wide(torch, eng, images, unary, G, p, potts=None, mus=None, between=None):
    """-> (Q_T, dL/dU (B, H, W, M), dL/dw (B, 2) or dL/dmu (B, 2, M, M) or None) from the two entry points; potts a
    (w1, w2) pair for the device weights, mus (mu_bi, mu_sp); `between(eng)` runs between forward and backward."""
    B, M = unary.shape[0], unary.shape[-1]
    u, g, im = _nchw(torch, unary), _nchw(torch, G), torch.from_numpy(images).cuda()
    q_hist = torch.empty((p.n_iters + 1,) + tuple(u.shape), device="cuda")
    gu = torch.empty_like(u)
    pt = None if potts is None else torch.tensor(potts, dtype=torch.float32, device="cuda")
    ct = None if mus is None else torch.from_numpy(np.stack(mus)).cuda()
    gp = torch.empty((B, 2), device="cuda") if mus is None else None
    gc = torch.empty((B, 2, M, M), device="cuda") if mus is not None else None
    eng.crf_forward_train_wide_dev(u, im, p, q_hist, potts=pt, compat=ct)
    if between is not None:
        between(eng)
    eng.crf_backward_wide_dev(q_hist, im, p, g, gu, potts=pt, compat=ct, grad_potts=gp, grad_compat=gc)
    torch.cuda.synchronize()
    return _nhwc(q_hist[p.n_iters]), _nhwc(gu), (gp if mus is None else gc).cpu().numpy()


def inputs(images, M, seed):
    B, H, W = images.shape[:3]
    unary = helpers.log_unary(B, H, W, M, seed, scale=1.0)
    return unary, np.stack([upstream(H, W, M, seed + b) for b in range(B)])


def check(torch, images, M, p, seed, potts=None, mus=None, eng=None, between=None):
    """Every image of the batch against its truth.  potts: device weights, which the truth takes through p."""
    B, H, W = images.shape[:3]
    unary, G = inputs(images, M, seed)
    eng = eng or api.Engine(B, H, W, M)
    tp = grad_params(p, p.n_iters, w1=potts[0], w2=potts[1]) if potts else p
    dev_p = grad_params(p, p.n_iters, w1=123.0, w2=-45.0) if potts else p   # the device weights must win
    q, gu, gparam = device_wide(torch, eng, images, unary, G, dev_p, potts, mus, between)
    for b in range(B):
        prob = meanfield64.Problem(images[b], tp)
        if mus is None:
            GradTruth(prob, unary[b], G[b], p.n_iters).check(gu[b], gparam[b], "image %d:" % b)
        else:
            CompatTruth(prob, unary[b], G[b], p.n_iters, mus).check(q[b], gu[b], gparam[b], "image %d:" % b)
    return eng


@pytest.mark.parametrize("M", WIDE_GRAD_M)
@pytest.mark.parametrize("kind", ["host", "device", "nonsym"])
def test_wide_grad_at_every_label_quad(torch_cuda, M, kind):
    """Phantom lanes at 33 (3 of 4 in the last quad) and 255 (1 of 4), whole quads at 36 and 128."""
    images = helpers.wide_images("smooth")
    p = grad_params(1.0, 2)
    check(torch_cuda, images, M, p, 40 + M, potts=(7.0, 2.5) if kind == "device" else None,
          mus=compat_mats("nonsym", M, M) if kind == "nonsym" else None)


@pytest.mark.parametrize("T", [0, 1, 2, 10])
@pytest.mark.parametrize("sf", [1.0, 12.0])
@pytest.mark.parametrize("kind", ["host", "nonsym"])
def test_wide_grad_at_every_iteration_count(torch_cuda, T, sf, kind):
    check(torch_cuda, helpers.wide_images("noise"), 33, grad_params(sf, T), 7 + T,
          mus=compat_mats("nonsym", 33, T) if kind == "nonsym" else None)


@pytest.mark.parametrize("img", ["smooth", "photo", "noise"])
@pytest.mark.parametrize("kind", ["device", "nonsym"])
def test_wide_grad_on_every_image_kind(torch_cuda, img, kind):
    images = np.stack([helpers.small_image(np.random.RandomState(51 + b), 23, 27, img) for b in range(2)])
    check(torch_cuda, images, 81, grad_params(1.0, 3), 11, potts=(10.0, 3.0) if kind == "device" else None,
          mus=compat_mats("nonsym", 81, 2) if kind == "nonsym" else None)


def test_training_forward_is_the_inference_forward(torch_cuda):
    """With host weights the training forward's q_hist[T] is dsrg_crf_batch_dev's result (the splat's atomics
    aside)."""
    torch = torch_cuda
    images = helpers.wide_images("noise")
    B, H, W = images.shape[:3]
    unary, _ = inputs(images, 81, 3)
    p = grad_params(1.0, 5)
    eng = api.Engine(B, H, W, 81)
    u, im = _nchw(torch, unary), torch.from_numpy(images).cuda()
    q_hist = torch.empty((6,) + tuple(u.shape), device="cuda")
    eng.crf_forward_train_wide_dev(u, im, p, q_hist)
    out = torch.empty_like(u)
    eng.crf_dev(u, im, p, out, unary_layout=api.LAYOUT_NCHW, out_layout=api.LAYOUT_NCHW)
    assert float((q_hist[5] - out).abs().max()) < 1e-5


def _slot_batch(problems, B):
    """Slot b: problem b % len(problems) with scale SCALES[b % 4]."""
    return [(b % len(problems), SCALES[b % len(SCALES)]) for b in range(B)]


def _scaled_check(truths, slots, gu, gparam, kind):
    for b, (pi, s) in enumerate(slots):
        t = truths[pi]
        e = float(np.abs(gu[b] - s * t.gU).max())
        assert e <= abs(s) * t.bar_u, "slot %d (problem %d, s %g): dL/dU off by %.3g > %.3g" % (
            b, pi, s, e, abs(s) * t.bar_u)
        if gparam is None:
            continue
        if kind == "potts":
            for i in (0, 1):
                ew = abs(float(gparam[b][i]) - s * t.gw[i])
                assert ew <= abs(s) * t.bar_w[i], "slot %d: dL/dw%d off by %.3g" % (b, i + 1, ew)
        else:
            d = np.abs(np.asarray(gparam[b], np.float64) - s * t.gmu) - abs(s) * t.bar_mu
            assert d.max() <= 0, "slot %d: dL/dmu off by %.3g beyond its bar" % (b, d.max())


def _problem_set(img, H, W, n, M, seed, p):
    images = np.stack([helpers.small_image(np.random.RandomState(seed + k), H, W, img) for k in range(n)])
    unary, G = inputs(images, M, seed)
    return images, unary, G, [meanfield64.Problem(images[k], p) for k in range(n)]


def _run_slots(torch, eng, probs, slots, p, mus=None, potts=None):
    images, unary, G, _ = probs
    idx = [pi for pi, _ in slots]
    s = np.array([sc for _, sc in slots], np.float32)[:, None, None, None]
    return device_wide(torch, eng, images[idx], unary[idx], (G[idx] * s).astype(np.float32), p, potts, mus)


@pytest.mark.parametrize("kind", ["potts", "nonsym"])
def test_slot_scaled_batches_and_engine_shapes(torch_cuda, kind):
    """Slot b holds problem pi(b) with upstream s_b G: a batch below the engine's, the engine's own, a re-shaped
    engine and back, and a spatial-sigma change (the shared spatial lattice rebuilt)."""
    torch = torch_cuda
    M = 81
    mus = compat_mats("nonsym", M, 5) if kind == "nonsym" else None
    eng = api.Engine(8, 41, 41, M)
    runs = [((41, 41), 12.0, 3), ((41, 41), 12.0, 8), ((19, 23), 1.0, 5), ((41, 41), 1.0, 8)]
    cache = {}
    for (H, W), sf, B in runs:
        p = grad_params(sf, 2)
        key = (H, W, sf)
        if key not in cache:
            probs = _problem_set("photo", H, W, 3, M, 61, p)
            images, unary, G, problems = probs
            cache[key] = (probs, [GradTruth(problems[k], unary[k], G[k], 2) if mus is None else
                                  CompatTruth(problems[k], unary[k], G[k], 2, mus) for k in range(3)])
        probs, truths = cache[key]
        eng.set_size(H, W)
        slots = _slot_batch(truths, B)
        _, gu, gparam = _run_slots(torch, eng, probs, slots, p, mus)
        _scaled_check(truths, slots, gu, gparam, kind)


def test_inference_between_forward_and_backward(torch_cuda):
    torch = torch_cuda
    images = helpers.wide_images("smooth")
    B, H, W = images.shape[:3]
    other = np.ascontiguousarray(images[::-1])

    def infer(eng):
        u = _nchw(torch, helpers.log_unary(B, H, W, 81, 99))
        out = torch.empty_like(u)
        eng.crf_dev(u, torch.from_numpy(other).cuda(), grad_params(12.0, 4), out, unary_layout=api.LAYOUT_NCHW,
                    out_layout=api.LAYOUT_NCHW)

    for mus in (None, compat_mats("nonsym", 81, 1)):
        check(torch, images, 81, grad_params(1.0, 3), 5, mus=mus, between=infer)


@pytest.mark.parametrize("name", sorted(GOLDEN_CASES))
def test_wide_grad_pinned_to_the_reference(torch_cuda, name):
    """The reference's own DenseCRF::gradient (frozen) and the device lie within the bar of the float64 truth."""
    image, unary, G, p, mus = golden_inputs(name)
    H, W, M = unary.shape
    q, gu, gparam = device_wide(torch_cuda, api.Engine(1, H, W, M), image[None], unary[None], G[None], p, mus=mus)
    prob = meanfield64.Problem(image, p)
    with np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", GOLDEN)) as z:
        if mus is None:
            t = GradTruth(prob, unary, G, p.n_iters)
            t.check(z[name + "/grad_unary"], (z[name + "/grad_w"][0], z[name + "/grad_w"][1]), "reference:")
        else:
            t = CompatTruth(prob, unary, G, p.n_iters, mus)
            t.check(z[name + "/q"], z[name + "/grad_unary"], None, "reference:")
    t.check(gu[0], gparam[0], "device:") if mus is None else t.check(q[0], gu[0], gparam[0], "device:")


@pytest.mark.parametrize("kind", ["potts", "nonsym"])
def test_coco_training_shape_through_dense_crf_wide(torch_cuda, kind):
    """Batch 20 @ 41x41, 81 labels, sf 12, T = 10 through nn.dense_crf_wide's autograd: every slot against s_b times
    its problem's truth (four problems)."""
    torch = torch_cuda
    M, B, T = 81, 20, 10
    p = grad_params(12.0, T)
    mus = compat_mats("nonsym", M, 9) if kind == "nonsym" else None
    images, unary, G, problems = _problem_set("photo", 41, 41, 4, M, 71, p)
    truths = [GradTruth(problems[k], unary[k], G[k], T) if mus is None else
              CompatTruth(problems[k], unary[k], G[k], T, mus) for k in range(4)]
    slots = _slot_batch(truths, B)
    idx = [pi for pi, _ in slots]
    s = np.array([sc for _, sc in slots], np.float32)[:, None, None, None]
    u = _nchw(torch, unary[idx]).requires_grad_(True)
    g = _nchw(torch, (G[idx] * s).astype(np.float32))
    im = torch.from_numpy(np.ascontiguousarray(images[idx])).cuda()
    if mus is None:
        w1 = torch.tensor(10.0, device="cuda", requires_grad=True)
        w2 = torch.tensor(3.0, device="cuda", requires_grad=True)
        out = nn.dense_crf_wide(u, im, 12.0, maxiter=T, w1=w1, w2=w2)
    else:
        cb = torch.from_numpy(mus[0]).cuda().requires_grad_(True)
        cs = torch.from_numpy(mus[1]).cuda().requires_grad_(True)
        out = nn.dense_crf_wide(u, im, 12.0, maxiter=T, compat_bi=cb, compat_sp=cs)
    (out * g).sum().backward()
    torch.cuda.synchronize()
    _scaled_check(truths, slots, _nhwc(u.grad), None, kind)
    # the parameters' gradients are the batch sums: sum_b s_b truth(pi(b)) under sum_b |s_b| bar(pi(b))
    if mus is None:
        for i, w in enumerate((w1, w2)):
            want = sum(sc * truths[pi].gw[i] for pi, sc in slots)
            bar = sum(abs(sc) * truths[pi].bar_w[i] for pi, sc in slots)
            assert abs(float(w.grad) - want) <= bar, "dL/dw%d %.9g, float64 %.9g" % (i + 1, float(w.grad), want)
    else:
        for k, c in enumerate((cb, cs)):
            want = sum(sc * truths[pi].gmu[k] for pi, sc in slots)
            bar = sum(abs(sc) * truths[pi].bar_mu[k] for pi, sc in slots)
            assert (np.abs(c.grad.cpu().numpy() - want) <= bar).all()


def test_one_321_photo_at_81_labels(torch_cuda):
    images = np.stack([helpers.small_image(np.random.RandomState(81), 321, 321, "photo")])
    check(torch_cuda, images, 81, grad_params(1.0, 2), 81, potts=(10.0, 3.0))


@pytest.mark.parametrize("kind", ["potts", "matrices"])
def test_captured_step_replayed_with_new_inputs(torch_cuda, kind):
    """One nn.dense_crf_wide step (forward + backward) captured in a CUDA graph and replayed after the unaries and the
    weights changed in place: the replay equals an eager step on the new values."""
    torch = torch_cuda
    images = helpers.wide_images("smooth")
    B, H, W = images.shape[:3]
    M = 81
    im = torch.from_numpy(images).cuda()
    g = _nchw(torch, inputs(images, M, 3)[1])
    u0 = _nchw(torch, inputs(images, M, 1)[0])
    u1 = _nchw(torch, inputs(images, M, 2)[0])
    if kind == "potts":
        params = [torch.tensor(v, device="cuda", requires_grad=True) for v in (10.0, 3.0)]
        new = [torch.tensor(v, device="cuda") for v in (6.0, 1.5)]
        kw = lambda ps: dict(w1=ps[0], w2=ps[1])
    else:
        params = [torch.from_numpy(m).cuda().requires_grad_(True) for m in compat_mats("nonsym", M, 2)]
        new = [torch.from_numpy(m).cuda() for m in compat_mats("nonsym", M, 3)]
        kw = lambda ps: dict(compat_bi=ps[0], compat_sp=ps[1])
    u = u0.clone().requires_grad_(True)

    def step():
        for t in [u] + params:
            t.grad = None
        (nn.dense_crf_wide(u, im, 1.0, maxiter=3, **kw(params)) * g).sum().backward()

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()   # warm up: the engine, its graphs and the backward's buffers
        graph = torch.cuda.CUDAGraph()
        for t in [u] + params:
            t.grad = None
        with torch.cuda.graph(graph, stream=s):
            (nn.dense_crf_wide(u, im, 1.0, maxiter=3, **kw(params)) * g).sum().backward()
    torch.cuda.current_stream().wait_stream(s)
    with torch.no_grad():
        u.copy_(u1)
        for p_, n_ in zip(params, new):
            p_.copy_(n_)
    graph.replay()
    torch.cuda.synchronize()
    got = [u.grad.clone()] + [p_.grad.clone() for p_ in params]
    ue = u1.clone().requires_grad_(True)
    pe = [n_.clone().requires_grad_(True) for n_ in new]
    (nn.dense_crf_wide(ue, im, 1.0, maxiter=3, **kw(pe)) * g).sum().backward()
    for a, b_ in zip(got, [ue.grad] + [p_.grad for p_ in pe]):
        assert torch.allclose(a, b_, rtol=1e-4, atol=1e-5), float((a - b_).abs().max())


def test_autocast(torch_cuda):
    torch = torch_cuda
    images = helpers.wide_images("noise")
    u = _nchw(torch, inputs(images, 40, 4)[0])
    im = torch.from_numpy(images).cuda()
    ref = nn.dense_crf_wide(u, im, maxiter=2)
    with torch.autocast("cuda", dtype=torch.float16):
        out = nn.dense_crf_wide(u.half(), im, maxiter=2)
    assert out.dtype == torch.float32
    assert float((out - ref).abs().max()) < 2e-3


def test_small_label_counts_are_dense_crf(torch_cuda):
    """At 32 labels or fewer dense_crf_wide is dense_crf: the same gradients up to the fused splat's float atomics."""
    torch = torch_cuda
    images = helpers.fused_images("smooth")
    u0 = _nchw(torch, inputs(images, 21, 6)[0])
    g = _nchw(torch, inputs(images, 21, 6)[1])
    im = torch.from_numpy(images).cuda()
    res = []
    for f in (nn.dense_crf, nn.dense_crf_wide):
        u = u0.clone().requires_grad_(True)
        w1 = torch.tensor(10.0, device="cuda", requires_grad=True)
        (f(u, im, maxiter=3, w1=w1) * g).sum().backward()
        res.append((u.grad, w1.grad))
    for a, b in zip(*res):
        assert torch.allclose(a, b, rtol=1e-5, atol=1e-6), float((a - b).abs().max())


def test_refusals_before_any_launch(torch_cuda):
    torch = torch_cuda
    images = helpers.wide_images("noise")
    B, H, W = images.shape[:3]
    im = torch.from_numpy(images).cuda()
    p = grad_params(1.0, 2)
    # the C pair refuses 32 labels and fewer, naming the fused pair
    small = api.Engine(B, H, W, 32)
    u = torch.zeros((B, 32, H, W), device="cuda")
    q = torch.empty((3, B, 32, H, W), device="cuda")
    small.take_launch_count()
    with pytest.raises(api.DsrgError) as e:
        small.crf_forward_train_wide_dev(u, im, p, q)
    assert e.value.code == _lib.E_INVALID and "dsrg_crf_forward_train_dev" in str(e.value)
    with pytest.raises(api.DsrgError) as e:
        small.crf_backward_wide_dev(q, im, p, u, torch.empty_like(u))
    assert e.value.code == _lib.E_INVALID
    assert small.take_launch_count() == 0
    # potts and compat together, grad_compat without compat
    eng = api.Engine(B, H, W, 40)
    u = torch.zeros((B, 40, H, W), device="cuda")
    q = torch.empty((3, B, 40, H, W), device="cuda")
    pt = torch.ones(2, device="cuda")
    ct = torch.zeros((2, 40, 40), device="cuda")
    eng.take_launch_count()
    with pytest.raises(api.DsrgError) as e:
        eng.crf_forward_train_wide_dev(u, im, p, q, potts=pt, compat=ct)
    assert e.value.code == _lib.E_INVALID
    with pytest.raises(api.DsrgError):
        eng.crf_backward_wide_dev(q, im, p, u, torch.empty_like(u), grad_compat=torch.empty((B, 2, 40, 40),
                                                                                           device="cuda"))
    assert eng.take_launch_count() == 0
    # nn.dense_crf_wide: every check before the first launch
    nn.dense_crf_wide(u, im, maxiter=2)   # creates the engine the refused calls would use
    torch.cuda.synchronize()
    eng = nn.cached_engine(40, H, W, torch.cuda.current_device())
    eng.take_launch_count()
    w = torch.tensor(1.0, device="cuda")
    bad = [dict(image=im[:1]), dict(image=im.float()), dict(w1=torch.ones(2, device="cuda")), dict(w1=1.0),
           dict(maxiter=-1), dict(w1=w, compat_bi=torch.zeros((40, 40), device="cuda")),
           dict(compat_sp=torch.zeros((39, 39), device="cuda"))]
    for kw in bad:
        args = dict(image=im, maxiter=2)
        args.update(kw)
        with pytest.raises(ValueError):
            nn.dense_crf_wide(u, args.pop("image"), **args)
    assert eng.take_launch_count() == 0
    # nn.dense_crf keeps its 32-label refusal and names dense_crf_wide
    with pytest.raises(ValueError, match="dense_crf_wide"):
        nn.dense_crf(u, im)
