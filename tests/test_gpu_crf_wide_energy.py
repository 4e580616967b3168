"""The CRF energy above 32 labels on the device (Engine.crf_energy_wide_dev / crf_energy_backward_wide_dev,
nn.dense_crf_energy_wide) against the float64 restatement (oracle/crf_energy_oracle.py, pinned to the reference's
klDivergence at 33 to 81 labels by test_crf_wide_energy_cpu.py): the terms and both gradients at 33 to 255 labels
under Potts weights (params' and the device's), matrices and caller-given features, at COCO's 81 labels on the
training shape and at 8 @ 321x321, the link to the fused path at 33 labels, autograd, CUDA graphs, the Potts / matrix
identity, the feature-range policy, the memory the first call takes, the refusals and the state.

Tolerance (crf_wide_energy_cases.energy_rel(M)): |device - truth| <= the worst-case float32 rounding of the
operations behind the value, counted from the label count, and never less than the fused path's 2^-16, times the sum
of the magnitudes behind the result."""
import numpy as np
import pytest

import helpers
from crf_compat_cases import compat_mats
from crf_energy_cases import grad_terms, problem, q_of
from crf_fgrad_cases import features_of
from crf_wide_energy_cases import check_grad, check_terms, energy_rel
from dsrg_b200 import _lib, api, synth
from oracle import crf_energy_oracle as E

pytestmark = pytest.mark.gpu


def _nchw(torch, a):
    return torch.from_numpy(np.ascontiguousarray(np.transpose(a, (0, 3, 1, 2)))).cuda()


def _hwc(t, b):
    return np.ascontiguousarray(np.transpose(t[b].detach().cpu().numpy(), (1, 2, 0)))


class Case(object):
    """One batch: images (B, H, W, 3), q and unary (B, M, H, W) on the device, params, the library's matrices or None,
    features (B, 5, H, W) or None, and the Potts weights as a device {w1, w2} or None."""

    def __init__(self, torch, B, H, W, img, sf, M, qkind, param, seed=0, q=None):
        if H >= 100:
            images = synth.make_batch(B, H, W, C=21, image=img, start=seed)["image"]
        else:
            images = np.stack([helpers.small_image(np.random.RandomState(seed + b), H, W, img) for b in range(B)])
        self.B, self.M, self.H, self.W = B, M, H, W
        self.images = images
        self.p = helpers.mf64_problem_params(sf, None, 0)
        self.image_d = torch.from_numpy(images).cuda()
        self.unary_np = helpers.log_unary(B, H, W, M, seed + 1, scale=1.0)
        self.unary = _nchw(torch, self.unary_np)
        if q is not None:
            self.q = q.contiguous()
        elif qkind == "softmax":
            self.q = torch.softmax(self.unary * 1.5, 1).contiguous()
        else:
            self.q = _nchw(torch, np.stack([q_of(qkind, H, W, M, seed + 11 + b) for b in range(B)]))
        self.mus = self.compat = self.feats = self.feats_d = self.potts = None
        if param == "matrix":
            self.mus = compat_mats("nonsym", M, seed + 2)
            self.compat = torch.from_numpy(np.stack(self.mus)).cuda()
        elif param == "features":
            self.feats = np.stack([features_of("guide", images[b], self.p, seed + b) for b in range(B)])
            self.feats_d = _nchw(torch, self.feats)
        elif param == "potts_dev":
            self.p.w1, self.p.w2 = 10.0, 3.0      # not used by the device: the kernels read `potts`
            self.potts = torch.tensor([6.5, 2.25], device="cuda")
        self.w = (6.5, 2.25) if param == "potts_dev" else (self.p.w1, self.p.w2)

    def engine(self, maxB=None):
        return api.Engine(maxB or self.B, self.H, self.W, self.M, device=0)

    def run(self, torch, eng, g=None, grad_unary=True, stream=None):
        """-> terms (B, 4) or, with g (B, 4), (grad_q, grad_unary)."""
        img = None if self.feats_d is not None else self.image_d
        kw = dict(features=self.feats_d, potts=self.potts, compat=self.compat, stream=stream)
        if g is None:
            terms = torch.full((self.B, 4), float("nan"), device="cuda")
            eng.crf_energy_wide_dev(self.q, self.unary, img, self.p, terms, **kw)
            return terms
        gq = torch.full_like(self.q, float("nan"))
        gu = torch.full_like(self.q, float("nan")) if grad_unary else None
        eng.crf_energy_backward_wide_dev(self.q, self.unary, img, self.p, torch.from_numpy(g).cuda(), gq, gu, **kw)
        return gq, gu

    def problem(self, b):
        p = helpers.mf64_problem_params(self.p, None, 0)
        p.w1, p.w2 = self.w
        return problem(self.images[b], p, None if self.feats is None else self.feats[b])

    def truth(self, b, g=None):
        P = self.problem(b)
        q = _hwc(self.q, b).astype(np.float64)
        if g is None:
            return E.terms(P, q, self.unary_np[b], self.mus)
        return E.gradient(P, q, self.unary_np[b], g[b], self.mus)

    def check(self, torch, eng, images, what=""):
        terms = self.run(torch, eng).cpu().numpy()
        g = grad_terms(self.B, 31)
        gq, gu = self.run(torch, eng, g)
        gq, gu = gq.cpu().numpy(), gu.cpu().numpy()
        for b in images:
            want, scale = self.truth(b)
            check_terms(terms[b], want, scale, self.M, "%s image %d" % (what, b))
            dq, du, sc = self.truth(b, g)
            check_grad(np.transpose(gq[b], (1, 2, 0)), dq, sc, self.M, "%s grad_q image %d" % (what, b))
            assert np.array_equal(np.transpose(gu[b], (1, 2, 0)), (-g[b, 1] * _hwc(self.q, b)).astype(np.float32)), \
                "%s grad_unary image %d" % (what, b)
        return terms


# ---- the label counts and the parameter kinds, at a small shape ----
@pytest.mark.parametrize("M", [33, 36, 37, 64, 81, 255])
@pytest.mark.parametrize("param", ["potts", "potts_dev", "matrix", "features"])
@pytest.mark.parametrize("qkind", ["random", "onehot"])
def test_label_counts_and_parameters(torch_cuda, M, param, qkind):
    torch = torch_cuda
    c = Case(torch, 2, 29, 37, "noise", 1.0, M, qkind, param, seed=M)
    c.check(torch, c.engine(), range(2), "M=%d %s %s" % (M, param, qkind))


# ---- COCO's 81 labels: the training shape on dense_crf_wide's marginals, and 8 @ 321x321 ----
def test_coco_train_shape_on_dense_crf_wide_marginals(torch_cuda):
    torch = torch_cuda
    from dsrg_b200 import nn
    c0 = Case(torch, 20, 41, 41, "smooth", 12.0, 81, "random", "potts_dev", seed=3)
    q = nn.dense_crf_wide(c0.unary, c0.image_d, scale_factor=12.0, maxiter=10)
    c = Case(torch, 20, 41, 41, "smooth", 12.0, 81, None, "potts_dev", seed=3, q=q)
    terms = c.check(torch, c.engine(), helpers.sample_indices(20, 5), "coco41")
    assert np.all(terms[:, 2:] < 0)   # Potts: every pairwise term is -w times a positive kernel mass


def test_coco_batch_8_at_321_one_hot_matrices(torch_cuda):
    torch = torch_cuda
    c = Case(torch, 8, 321, 321, "photo", 1.0, 81, "onehot", "matrix", seed=40)
    c.check(torch, c.engine(), [0, 7], "8@321")


# ---- the link to the fused path: a 33rd label with zero q, unary and matrix entries changes nothing ----
@pytest.mark.parametrize("param", ["potts_dev", "matrix"])
def test_33_labels_with_an_empty_label_equal_the_fused_32(torch_cuda, param):
    torch = torch_cuda
    c32 = Case(torch, 2, 29, 37, "photo", 1.0, 32, "random", param, seed=50)
    c33 = Case(torch, 2, 29, 37, "photo", 1.0, 33, "random", param, seed=50)
    pad = lambda t: torch.cat([t, torch.zeros_like(t[:, :1])], 1).contiguous()
    c33.q, c33.unary = pad(c32.q), pad(c32.unary)
    if param == "matrix":
        c33.compat = torch.zeros((2, 33, 33), device="cuda")
        c33.compat[:, :32, :32] = c32.compat
    g = grad_terms(2, 9)
    eng32 = c32.engine()   # the fused energy, dsrg_crf_energy_dev
    t32 = torch.full((2, 4), float("nan"), device="cuda")
    gq32 = torch.full_like(c32.q, float("nan"))
    kw = dict(potts=c32.potts, compat=c32.compat)
    eng32.crf_energy_dev(c32.q, c32.unary, c32.image_d, c32.p, t32, **kw)
    eng32.crf_energy_backward_dev(c32.q, c32.unary, c32.image_d, c32.p, torch.from_numpy(g).cuda(), gq32, **kw)
    eng33 = c33.engine()
    t33 = c33.run(torch, eng33).cpu().numpy()
    gq33 = c33.run(torch, eng33, g)[0].cpu().numpy()
    t32, gq32 = t32.cpu().numpy(), gq32.cpu().numpy()
    for b in range(2):
        _, scale = c32.truth(b)
        assert np.all(np.abs(t33[b] - t32[b]) <= energy_rel(33) * scale), (t33[b], t32[b])
        _, _, sc = c32.truth(b, g)
        assert np.all(np.abs(gq33[b, :32] - gq32[b]) <= energy_rel(33) * np.transpose(sc, (2, 0, 1)))


# ---- Potts = matrices at mu = -w I ----
def test_potts_call_equals_matrix_call(torch_cuda):
    torch = torch_cuda
    M = 81
    c = Case(torch, 3, 41, 41, "noise", 1.0, M, "random", "potts_dev", seed=14)
    eng = c.engine()
    g = grad_terms(3, 6)
    t_p = c.run(torch, eng).cpu().numpy()
    gq_p = c.run(torch, eng, g)[0].cpu().numpy()
    eye = np.eye(M, dtype=np.float32)
    c.potts, c.compat = None, torch.from_numpy(np.stack([-6.5 * eye, -2.25 * eye])).cuda()
    t_m = c.run(torch, eng).cpu().numpy()
    gq_m = c.run(torch, eng, g)[0].cpu().numpy()
    # the same products (mu's zeros add exactly); the splats' float atomics may add in another order
    assert np.all(np.abs(t_p - t_m) <= 2.0 ** -20 * np.abs(t_p) + 1e-3), (t_p, t_m)
    assert np.all(np.abs(gq_p - gq_m) <= 2.0 ** -18 * np.abs(gq_p).max())


# ---- autograd ----
@pytest.mark.parametrize("param", ["potts", "matrix", "features"])
def test_autograd_through_dense_crf_energy_wide(torch_cuda, param):
    torch = torch_cuda
    from dsrg_b200 import nn
    M = 81
    c = Case(torch, 2, 29, 37, "photo", 1.0, M, "softmax", param, seed=8)
    q = c.q.clone().requires_grad_()
    u = c.unary.clone().requires_grad_()
    kw = {}
    if param == "matrix":
        kw = dict(compat_bi=c.compat[0], compat_sp=c.compat[1])
    elif param == "features":
        kw = dict(features_bi=c.feats_d)
    img = None if param == "features" else c.image_d
    with torch.autocast("cuda", dtype=torch.bfloat16):   # the layer casts to float32 and computes in it
        terms = nn.dense_crf_energy_wide(q, u, img, **kw)
    assert terms.dtype == torch.float32 and tuple(terms.shape) == (2, 4)
    g = grad_terms(2, 17)
    (terms * torch.from_numpy(g).cuda()).sum().backward()
    for b in range(2):
        want, scale = c.truth(b)
        check_terms(terms[b].detach().cpu().numpy(), want, scale, M, "autograd image %d" % b)
        dq, du, sc = c.truth(b, g)
        check_grad(_hwc(q.grad, b), dq, sc, M, "autograd grad_q image %d" % b)
        assert np.allclose(_hwc(u.grad, b), du, rtol=1e-6, atol=0)
    q2 = c.q.clone().requires_grad_()   # no unary: its term is 0 and q still gets the gradient
    t2 = nn.dense_crf_energy_wide(q2, None, img, **kw)
    assert np.all(t2[:, 1].detach().cpu().numpy() == 0.0)
    t2[:, 2:].sum().backward()
    assert torch.isfinite(q2.grad).all()
    c.unary_np = np.zeros_like(c.unary_np)
    for b in range(2):
        dq, _, sc = c.truth(b, np.array([[0.0, 0.0, 1.0, 1.0]] * 2))
        check_grad(_hwc(q2.grad, b), dq, sc, M, "no-unary grad_q image %d" % b)


def test_dense_crf_energy_wide_is_dense_crf_energy_at_32_labels_or_fewer(torch_cuda):
    torch = torch_cuda
    from dsrg_b200 import nn
    c = Case(torch, 2, 29, 37, "photo", 1.0, 21, "softmax", "matrix", seed=18)
    kw = dict(compat_bi=c.compat[0], compat_sp=c.compat[1])
    outs = []
    for f in (nn.dense_crf_energy, nn.dense_crf_energy_wide):
        q = c.q.clone().requires_grad_()
        u = c.unary.clone().requires_grad_()
        t = f(q, u, c.image_d, **kw)
        (t * torch.from_numpy(grad_terms(2, 4)).cuda()).sum().backward()
        outs.append([x.detach().cpu().numpy() for x in (t, q.grad, u.grad)])
    (t1, gq1, gu1), (t2, gq2, gu2) = outs
    for b in range(2):
        _, scale = c.truth(b)
        # one path, run twice: the splats' float atomics are the only difference
        assert np.all(np.abs(t1[b] - t2[b]) <= 2.0 ** -20 * scale), (t1[b], t2[b])
    assert np.all(np.abs(gq1 - gq2) <= 2.0 ** -18 * np.abs(gq1).max())
    assert np.array_equal(gu1, gu2)


# ---- graphs: a caller's capture and the engine's own replays ----
def test_cuda_graph_replay_equals_the_eager_call(torch_cuda):
    torch = torch_cuda
    M = 81
    c = Case(torch, 4, 41, 41, "photo", 12.0, M, "softmax", "matrix", seed=12)
    eng = c.engine()
    g = grad_terms(4, 3)
    c.run(torch, eng)                                   # the first call allocates: outside the capture
    c.run(torch, eng, g)
    torch.cuda.synchronize()
    terms = torch.empty(4, 4, device="cuda")
    gq = torch.empty_like(c.q)
    gt = torch.from_numpy(g).cuda()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        eng.crf_energy_wide_dev(c.q, c.unary, c.image_d, c.p, terms, compat=c.compat)
        eng.crf_energy_backward_wide_dev(c.q, c.unary, c.image_d, c.p, gt, gq, compat=c.compat)
    new_q = torch.softmax(torch.randn_like(c.q) * 2.0, 1)
    c.q.copy_(new_q)                                    # values change, addresses do not
    graph.replay()
    torch.cuda.synchronize()
    eager_t = c.run(torch, eng).cpu().numpy()
    eager_g = c.run(torch, eng, g)[0].cpu().numpy()
    got_t, got_g = terms.cpu().numpy(), gq.cpu().numpy()
    for b in range(4):
        want, scale = c.truth(b)
        check_terms(got_t[b], want, scale, M, "replay image %d" % b)
        # the splat adds with float atomics in no fixed order: replay and eager agree to that rounding
        assert np.all(np.abs(got_t[b] - eager_t[b]) <= 2.0 ** -20 * scale), (got_t[b], eager_t[b])
        _, _, sc = c.truth(b, g)
        assert np.all(np.abs(got_g[b] - eager_g[b]) <= 2.0 ** -20 * np.transpose(sc, (2, 0, 1)))
    # the engine's own graph: the third call on a side stream replays the second's capture
    s = torch.cuda.Stream()
    terms2 = torch.empty(4, 4, device="cuda")
    gq2 = torch.empty_like(c.q)
    torch.cuda.synchronize()
    outs = []
    with torch.cuda.stream(s):
        before = eng.graph_replays
        for _ in range(3):
            eng.crf_energy_wide_dev(c.q, c.unary, c.image_d, c.p, terms2, compat=c.compat)
            outs.append(terms2.cpu().numpy())
        assert eng.graph_replays > before
        before = eng.graph_replays
        for _ in range(3):
            eng.crf_energy_backward_wide_dev(c.q, c.unary, c.image_d, c.p, gt, gq2, compat=c.compat)
        assert eng.graph_replays > before
        got_g2 = gq2.cpu().numpy()
    for o in outs:
        assert np.all(np.abs(o - eager_t) <= 2.0 ** -20 * np.abs(eager_t) + 1e-3), (o, eager_t)
    assert np.all(np.abs(got_g2 - eager_g) <= 2.0 ** -18 * np.abs(eager_g).max())


# ---- features out of range: NaN for that image only ----
def test_out_of_range_features_give_nan_for_that_image_only(torch_cuda):
    torch = torch_cuda
    M = 40
    c = Case(torch, 3, 29, 37, "photo", 1.0, M, "random", "features", seed=20)
    c.feats = c.feats.copy()
    c.feats[1] *= 400.0
    c.feats_d = _nchw(torch, c.feats)
    eng = c.engine()
    g = grad_terms(3, 2)
    terms = c.run(torch, eng).cpu().numpy()
    assert list(eng.feature_range_flags(3)) == [False, True, False]
    gq, gu = c.run(torch, eng, g)
    assert list(eng.feature_range_flags(3)) == [False, True, False]
    gq, gu = gq.cpu().numpy(), gu.cpu().numpy()
    assert np.all(np.isnan(terms[1])) and np.all(np.isnan(gq[1])) and np.all(np.isnan(gu[1]))
    for b in (0, 2):
        want, scale = c.truth(b)
        check_terms(terms[b], want, scale, M, "image %d" % b)
        dq, _, sc = c.truth(b, g)
        check_grad(np.transpose(gq[b], (1, 2, 0)), dq, sc, M, "image %d" % b)


# ---- a batch smaller than the engine's ----
def test_batch_below_the_engine_capacity(torch_cuda):
    torch = torch_cuda
    c = Case(torch, 2, 29, 37, "smooth", 1.0, 81, "softmax", "matrix", seed=22)
    c.check(torch, c.engine(maxB=5), range(2), "B=2 of 5")


# ---- memory, state and refusals ----
@pytest.mark.parametrize("B,H,W,want", [(20, 41, 41, 4480), (8, 321, 321, 103168)])
def test_first_call_allocates_the_block_sums(torch_cuda, B, H, W, want):
    torch = torch_cuda
    M = 81
    eng = api.Engine(B, H, W, M, device=0)
    assert want == B * -(-H * W // 256) * 32
    q = torch.full((1, M, H, W), 1.0 / M, device="cuda")
    image = torch.zeros((1, H, W, 3), dtype=torch.uint8, device="cuda")
    terms = torch.empty(1, 4, device="cuda")
    p = api.crf_params(12.0, 13, 0)
    before = eng.device_bytes
    eng.crf_energy_wide_dev(q, None, image, p, terms)
    assert eng.device_bytes - before == want
    eng.crf_energy_backward_wide_dev(q, None, image, p, torch.ones(1, 4, device="cuda"), torch.empty_like(q))
    assert eng.device_bytes - before == want
    torch.cuda.synchronize()
    # a constant q: the entropy is N log(1/M), and there is no unary term
    assert abs(terms[0, 0].item() - H * W * np.log(np.float32(1.0 / M))) <= 1e-5 * H * W * np.log(M)
    assert terms[0, 1].item() == 0.0


def test_refusals_state_and_profile(torch_cuda):
    torch = torch_cuda
    H, W = 8, 8
    image = torch.zeros((1, H, W, 3), dtype=torch.uint8, device="cuda")
    p = api.crf_params(1.0, 13, 0)
    for M in (21, 32):   # the fused pair serves 32 labels or fewer
        q = torch.full((1, M, H, W), 0.1, device="cuda")
        fused = api.Engine(1, H, W, M, device=0)
        before = fused.device_bytes
        for call in (lambda: fused.crf_energy_wide_dev(q, None, image, p, torch.empty(1, 4, device="cuda")),
                     lambda: fused.crf_energy_backward_wide_dev(q, None, image, p, torch.ones(1, 4, device="cuda"),
                                                                torch.empty_like(q))):
            with pytest.raises(_lib.DsrgError) as ei:
                call()
            assert ei.value.code == -1 and "more than 32" in str(ei.value)
        assert fused.device_bytes == before
    M = 40
    eng = api.Engine(1, H, W, M, device=0)
    q = torch.full((1, M, H, W), 0.1, device="cuda")
    f = torch.zeros((1, 5, H, W), device="cuda")
    terms = torch.empty(1, 4, device="cuda")
    potts = torch.tensor([1.0, 1.0], device="cuda")
    compat = torch.zeros((2, M, M), device="cuda")
    before = eng.device_bytes
    for kw in (dict(image=image, features=f), dict(image=None), dict(image=image, potts=potts, compat=compat)):
        img = kw.pop("image")
        with pytest.raises(_lib.DsrgError) as ei:
            eng.crf_energy_wide_dev(q, None, img, p, terms, **kw)
        assert ei.value.code == -1
        with pytest.raises(_lib.DsrgError) as ei:
            eng.crf_energy_backward_wide_dev(q, None, img, p, torch.ones(1, 4, device="cuda"), torch.empty_like(q),
                                             **kw)
        assert ei.value.code == -1
    assert eng.device_bytes == before
    # an energy call leaves no marginals for the *_last_* entry points
    eng.crf_dev(torch.zeros((1, H, W, M), device="cuda"), image, api.crf_params(1.0), torch.empty((1, H, W, M),
                                                                                                   device="cuda"))
    eng.crf_energy_wide_dev(q, None, image, p, terms)
    with pytest.raises(_lib.DsrgError) as ei:
        eng.srg_last_crf_dev(torch.ones((1, M), device="cuda"), torch.zeros_like(q), 0.99, 0.85, torch.empty_like(q))
    assert ei.value.code == -4
    for call in (lambda: eng.crf_energy_wide_dev(q, None, image, p, terms, compat=compat),
                 lambda: eng.crf_energy_backward_wide_dev(q, None, image, p, torch.ones(1, 4, device="cuda"),
                                                          torch.empty_like(q), compat=compat)):
        eng.profile(True)
        call()
        prof = eng.profile_read()
        eng.profile(False)
        assert prof["crf_energy"][1] >= 10
        assert not any(k.startswith("mf_") or k in ("wide_grad", "kernel_grad", "feature_grad") for k in prof), prof
