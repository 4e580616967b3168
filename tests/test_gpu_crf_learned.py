"""The learned CRF at inference on the device (nn.dense_crf_inference, Engine.crf_learned_dev,
Engine.predict_mask_batch_learned_dev and the learned keywords of postprocess.predict_mask_batch_dev /
predict_masks_dev) against dense_crf / dense_crf_wide's training forward, the float64 restatements, the reference's
MatrixCompatibility (frozen), and the Potts inference at the identities mu = -w I and features = the image's own;
memory, graphs, the feature-range policy and the refusals."""
import ctypes as C
import os

import numpy as np
import pytest

import helpers
from crf_compat_cases import GOLDEN, GOLDEN_CASES, compat_mats, golden_inputs
from dsrg_b200 import _lib, api
from oracle import crf_compat_oracle, crf_fgrad_oracle, meanfield64

pytestmark = pytest.mark.gpu

BOUND = 1e-4   # the project's CRF bound (max abs on marginals)


def _nchw(torch, a):
    return torch.from_numpy(np.ascontiguousarray(np.transpose(a, (0, 3, 1, 2)))).cuda()


def _inputs(torch, M, B=2, H=29, W=37, img="noise", seed=3):
    rng = np.random.RandomState(seed)
    images = np.stack([helpers.small_image(rng, H, W, img) for _ in range(B)])
    unary = helpers.log_unary(B, H, W, M, seed)
    return torch.from_numpy(images).cuda(), _nchw(torch, unary)


def _features(torch, image, p):
    """The image's own bilateral features (B, 5, H, W), as the image path computes them."""
    f = np.stack([crf_fgrad_oracle.image_features(im, p) for im in image.cpu().numpy()])
    return _nchw(torch, f)


def _mats(torch, kind, M, seed=1):
    return [torch.from_numpy(m).cuda() for m in compat_mats(kind, M, seed)]


def _scalar(torch, v):
    return torch.tensor(float(v), device="cuda")


# ---- against the training forward, with the same arguments ----
KINDS = ["weights", "sym", "nonsym", "theta", "features", "features_theta_sp", "features_nonsym"]


@pytest.mark.parametrize("M", [1, 2, 21, 32, 33, 81])
@pytest.mark.parametrize("kind", KINDS)
def test_matches_the_training_forward(torch_cuda, M, kind):
    torch = torch_cuda
    from dsrg_b200 import nn
    image, unary = _inputs(torch, M, seed=M)
    kw = {}
    if kind == "weights":
        kw = dict(w1=_scalar(torch, 6.5), w2=_scalar(torch, 2.0))
    elif kind in ("sym", "nonsym"):
        kw["compat_bi"], kw["compat_sp"] = _mats(torch, kind, M)
    elif kind == "theta":
        kw = dict(theta_bi=torch.tensor([70.0, 90.0, 11.0, 14.0, 12.0]), theta_sp=torch.tensor([2.5, 3.5]))
    if kind.startswith("features"):
        kw["features_bi"] = _features(torch, image, api.crf_params(1.0)) * 0.8
        if kind == "features_theta_sp":
            kw["theta_sp"] = torch.tensor([2.0, 4.0])
        if kind == "features_nonsym":
            kw["compat_bi"], kw["compat_sp"] = _mats(torch, "nonsym", M, 2)
        img = None
    else:
        img = image
    with torch.no_grad():
        want = nn.dense_crf_wide(unary, img, **kw)
    got = nn.dense_crf_inference(unary, img, **kw)
    torch.cuda.synchronize()
    err = float((got - want).abs().max())
    print("M=%d %s: max |inference - training forward| = %.3g" % (M, kind, err))
    assert err <= BOUND
    assert not got.requires_grad


# ---- against the float64 restatements and the reference ----
@pytest.mark.parametrize("M,kind", [(6, "sym"), (21, "nonsym"), (33, "sym")])
def test_matrices_match_the_float64_restatement(torch_cuda, M, kind):
    torch = torch_cuda
    from dsrg_b200 import nn
    image, unary = _inputs(torch, M, B=1, H=23, W=31, seed=7)
    mus = compat_mats(kind, M, 4)
    got = nn.dense_crf_inference(unary, image, compat_bi=torch.from_numpy(mus[0]).cuda(),
                                 compat_sp=torch.from_numpy(mus[1]).cuda())
    p = api.crf_params(1.0)
    want = crf_compat_oracle.run(meanfield64.Problem(image[0].cpu().numpy(), p),
                                 np.transpose(unary[0].cpu().numpy(), (1, 2, 0)), mus, 10)[10]
    err = float(np.abs(np.transpose(got[0].cpu().numpy(), (1, 2, 0)) - want).max())
    print("M=%d %s: max |device - float64| = %.3g" % (M, kind, err))
    assert err <= BOUND


@pytest.mark.parametrize("M", [5, 40])
def test_features_match_the_float64_restatement(torch_cuda, M):
    torch = torch_cuda
    from dsrg_b200 import nn
    image, unary = _inputs(torch, M, B=1, H=21, W=27, seed=9)
    p = api.crf_params(1.0)
    f = crf_fgrad_oracle.image_features(image[0].cpu().numpy(), p) * np.float32(0.7)
    got = nn.dense_crf_inference(unary, None, features_bi=_nchw(torch, f[None]))
    want = crf_fgrad_oracle.FeatProblem(f, p).run(np.transpose(unary[0].cpu().numpy(), (1, 2, 0)), 10)[10]
    err = float(np.abs(np.transpose(got[0].cpu().numpy(), (1, 2, 0)) - want).max())
    print("M=%d: max |device - float64| = %.3g" % (M, err))
    assert err <= BOUND


@pytest.mark.parametrize("name", sorted(GOLDEN_CASES))
def test_matrices_match_the_reference(torch_cuda, name):
    """The reference's own MatrixCompatibility inference (frozen in the golden file's /q)."""
    torch = torch_cuda
    from dsrg_b200 import nn
    image, unary, _, p, mus = golden_inputs(name)
    sf = GOLDEN_CASES[name][4]
    got = nn.dense_crf_inference(_nchw(torch, unary[None]), torch.from_numpy(image[None]).cuda(), scale_factor=sf,
                                 maxiter=p.n_iters, compat_bi=torch.from_numpy(mus[0]).cuda(),
                                 compat_sp=torch.from_numpy(mus[1]).cuda())
    with np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", GOLDEN)) as z:
        want = z[name + "/q"]
    err = float(np.abs(np.transpose(got[0].cpu().numpy(), (1, 2, 0)) - want).max())
    print("%s: max |device - reference| = %.3g" % (name, err))
    assert err <= BOUND


# ---- identities against the Potts inference (dsrg_crf_batch_dev) ----
@pytest.mark.parametrize("M", [21, 81])
@pytest.mark.parametrize("kind", ["potts_matrices", "image_features"])
def test_identities_against_the_potts_inference(torch_cuda, M, kind):
    torch = torch_cuda
    image, unary = _inputs(torch, M, B=3, H=41, W=53, img="photo" if M == 21 else "noise", seed=M)
    B, _, H, W = unary.shape
    eng = api.Engine(B, H, W, M)
    p = api.crf_params(1.0)
    want = torch.empty_like(unary)
    eng.crf_dev(unary, image, p, want, api.LAYOUT_NCHW, api.LAYOUT_NCHW)
    got = torch.empty_like(unary)
    if kind == "potts_matrices":
        compat = torch.stack([-p.w1 * torch.eye(M, device="cuda"), -p.w2 * torch.eye(M, device="cuda")]).contiguous()
        eng.crf_learned_dev(unary, image, p, got, compat=compat, unary_layout=api.LAYOUT_NCHW,
                            out_layout=api.LAYOUT_NCHW)
    else:
        eng.crf_learned_dev(unary, None, p, got, features=_features(torch, image, p), unary_layout=api.LAYOUT_NCHW,
                            out_layout=api.LAYOUT_NCHW)
    torch.cuda.synchronize()
    err = float((got - want).abs().max())
    print("M=%d %s: max |learned - Potts| = %.3g" % (M, kind, err))
    assert err <= BOUND


# ---- predict_mask with the learned CRF at those identities ----
def _post_inputs(torch, B, H, W, M, seed):
    rng = np.random.RandomState(seed)
    images = torch.from_numpy(np.stack([helpers.small_image(rng, H, W, "photo") for _ in range(B)])).cuda()
    scores = [torch.from_numpy(rng.randn(B, M, h, w).astype(np.float32) * 3).cuda() for h, w in ((9, 11), (13, 15))]
    tags = torch.from_numpy((rng.rand(B, M) > 0.7).astype(np.float32)).cuda()
    return images, scores, tags


def _sure(probs, bound=2e-4):
    top2 = probs.topk(2, dim=-1).values
    return (top2[..., 0] - top2[..., 1]) > bound


@pytest.mark.parametrize("M", [21, 81])
@pytest.mark.parametrize("mode", ["ms", "gt"])
@pytest.mark.parametrize("kind", ["potts_matrices", "image_features"])
def test_predict_mask_identities(torch_cuda, M, mode, kind):
    torch = torch_cuda
    B, H, W = 3, 47, 61
    images, scores, tags = _post_inputs(torch, B, H, W, M, M + 1)
    if mode == "gt":
        scores = scores[:1]
    eng = api.Engine(B, H, W, M)
    p = api.crf_params(1.0)
    sel = None
    if mode == "gt":
        present = tags > 0.5
        present[:, 0] = True
        ids = torch.arange(M, device="cuda", dtype=torch.int32).expand(B, M)
        order = torch.sort(torch.where(present, ids, ids + M), dim=1).values
        sel = torch.where(order < M, order, torch.full_like(order, -1)).contiguous()
    md = api.POST_SUM_SCORES if mode == "ms" else api.POST_ZOOM_PROBS
    want_l = torch.empty((B, H, W), dtype=torch.int32, device="cuda")
    want_p = torch.empty((B, H, W, M), dtype=torch.float32, device="cuda")
    eng.predict_mask_batch_dev(scores, images, want_l, p, md, sel=sel, probs_out=want_p)
    got_l, got_p = torch.empty_like(want_l), torch.empty_like(want_p)
    if kind == "potts_matrices":
        compat = torch.stack([-p.w1 * torch.eye(M, device="cuda"), -p.w2 * torch.eye(M, device="cuda")]).contiguous()
        eng.predict_mask_batch_learned_dev(scores, images, got_l, p, md, compat=compat, sel=sel, probs_out=got_p)
    else:
        eng.predict_mask_batch_learned_dev(scores, None, got_l, p, md, features=_features(torch, images, p), sel=sel,
                                           probs_out=got_p)
    torch.cuda.synchronize()
    err = float((got_p - want_p).abs().max())
    print("M=%d %s %s: max |probs - Potts path| = %.3g" % (M, mode, kind, err))
    assert err <= BOUND
    sure = _sure(want_p)
    assert torch.equal(got_l[sure], want_l[sure])


def _engine_reference(torch, images, scores, M, mode=api.POST_SUM_SCORES):
    """Today's path, CRF()'s CRF: (label maps, probabilities) from Engine.predict_mask_batch_dev with probs_out."""
    B, H, W = images.shape[:3]
    eng = api.Engine(B, H, W, M)
    lab = torch.empty((B, H, W), dtype=torch.int32, device="cuda")
    probs = torch.empty((B, H, W, M), dtype=torch.float32, device="cuda")
    eng.predict_mask_batch_dev(scores, images, lab, api.crf_params(1.0), mode, probs_out=probs)
    torch.cuda.synchronize()
    eng.close()
    return lab, probs


def test_postprocess_keywords_at_the_identities(torch_cuda):
    """predict_mask_batch_dev(compat_bi=-w1 I, compat_sp=-w2 I), and predict_masks_dev on mixed VOC sizes with
    per-image features: every image's label map equals today's wherever today's top two marginals are 2e-4 apart, so a
    group's images, scores and features stay aligned through the grouping."""
    torch = torch_cuda
    from dsrg_b200 import postprocess
    M = 21
    p = api.crf_params(1.0)
    images, scores, _ = _post_inputs(torch, 2, 45, 57, M, 5)
    eye = torch.eye(M, device="cuda")
    want_l, want_p = _engine_reference(torch, images, scores, M)
    got = postprocess.predict_mask_batch_dev(images, scores, compat_bi=-p.w1 * eye, compat_sp=-p.w2 * eye)
    torch.cuda.synchronize()
    sure = _sure(want_p)
    assert torch.equal(got[sure], want_l[sure])
    rng = np.random.RandomState(8)
    sizes = [(375, 500), (500, 375), (375, 500), (333, 500)]
    ims = [torch.from_numpy(helpers.small_image(rng, h, w, "photo")).cuda() for h, w in sizes]
    sc = [torch.from_numpy(rng.randn(len(ims), M, 41, 41).astype(np.float32) * 3).cuda()]
    feats = [_features(torch, im[None], p)[0] for im in ims]
    got = postprocess.predict_masks_dev(ims, sc, mode="ms", features_bi=feats)
    torch.cuda.synchronize()
    for i, g in enumerate(got):
        want_l, want_p = _engine_reference(torch, ims[i][None].contiguous(), [sc[0][i:i + 1].contiguous()], M)
        sure = _sure(want_p[0])
        assert torch.equal(g[sure], want_l[0][sure]), i


# ---- memory ----
def test_memory_keeps_no_history(torch_cuda):
    torch = torch_cuda
    from dsrg_b200 import nn
    M = 21
    image, unary = _inputs(torch, M, B=4, H=64, W=80, seed=2)
    compat = _mats(torch, "sym", M)
    nn.dense_crf_inference(unary, image, compat_bi=compat[0], compat_sp=compat[1])   # the engine exists now
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = nn.dense_crf_inference(unary, image, compat_bi=compat[0], compat_sp=compat[1])
    torch.cuda.synchronize()
    grew = torch.cuda.max_memory_allocated() - base
    print("peak growth %d bytes, output %d bytes" % (grew, out.numel() * 4))
    assert grew <= out.numel() * 4 + 4096   # the output (rounded to the allocator's block) and nothing per iteration


def test_device_bytes_grow_by_the_feature_flags_only(torch_cuda):
    torch = torch_cuda
    for M in (21, 81):
        image, unary = _inputs(torch, M, B=2, H=33, W=41, seed=M)
        B, _, H, W = unary.shape
        eng = api.Engine(B, H, W, M)
        p = api.crf_params(1.0)
        out = torch.empty_like(unary)
        b0 = eng.device_bytes
        eng.crf_learned_dev(unary, image, p, out, unary_layout=api.LAYOUT_NCHW, out_layout=api.LAYOUT_NCHW)
        assert eng.device_bytes == b0                  # Potts: nothing
        eng.crf_learned_dev(unary, None, p, out, features=_features(torch, image, p), unary_layout=api.LAYOUT_NCHW,
                            out_layout=api.LAYOUT_NCHW)
        b1 = eng.device_bytes
        assert b1 - b0 <= 64                           # the per-image key-range flags
        compat = torch.stack(_mats(torch, "sym", M)).contiguous()
        eng.crf_learned_dev(unary, image, p, out, compat=compat, unary_layout=api.LAYOUT_NCHW,
                            out_layout=api.LAYOUT_NCHW)
        b2 = eng.device_bytes
        assert b2 == b1                                # matrices: nothing, at every label count
        eng.crf_learned_dev(unary, image, p, out, compat=compat, unary_layout=api.LAYOUT_NCHW,
                            out_layout=api.LAYOUT_NCHW)
        assert eng.device_bytes == b2
        torch.cuda.synchronize()
        eng.close()


# ---- graphs ----
@pytest.mark.parametrize("M", [21, 33])
def test_replays_follow_in_place_edits(torch_cuda, M):
    torch = torch_cuda
    from dsrg_b200 import nn
    image, unary = _inputs(torch, M, B=2, H=31, W=39, seed=4)
    B, _, H, W = unary.shape
    eng = api.Engine(B, H, W, M)
    p = api.crf_params(1.0)
    compat = torch.stack(_mats(torch, "nonsym", M)).contiguous()
    feats = _features(torch, image, p)
    out = torch.empty_like(unary)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for _ in range(2):
            eng.crf_learned_dev(unary, None, p, out, features=feats, compat=compat, unary_layout=api.LAYOUT_NCHW,
                                out_layout=api.LAYOUT_NCHW, stream=s.cuda_stream)
        r0 = eng.graph_replays
        compat.mul_(0.5)
        feats.mul_(1.3)
        eng.crf_learned_dev(unary, None, p, out, features=feats, compat=compat, unary_layout=api.LAYOUT_NCHW,
                            out_layout=api.LAYOUT_NCHW, stream=s.cuda_stream)
    s.synchronize()
    assert eng.graph_replays > r0
    with torch.no_grad():
        want = nn.dense_crf_wide(unary, None, compat_bi=compat[0], compat_sp=compat[1], features_bi=feats)
    assert float((out - want).abs().max()) <= BOUND


def test_captured_in_a_torch_graph(torch_cuda):
    torch = torch_cuda
    from dsrg_b200 import nn
    M = 21
    image, unary = _inputs(torch, M, B=2, H=31, W=39, seed=6)
    compat = torch.stack(_mats(torch, "sym", M)).contiguous()
    feats = _features(torch, image, api.crf_params(1.0))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        nn.dense_crf_inference(unary, None, compat_bi=compat[0], compat_sp=compat[1], features_bi=feats)
    torch.cuda.current_stream().wait_stream(s)
    w1 = _scalar(torch, 5.0)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = nn.dense_crf_inference(unary, None, compat_bi=compat[0], compat_sp=compat[1], features_bi=feats)
        with pytest.raises(ValueError, match="CUDA-graph capture"):
            nn.dense_crf_inference(unary, image, theta_sp=torch.tensor([2.0, 2.0]))
        with pytest.raises(ValueError, match="CUDA-graph capture"):
            nn.dense_crf_inference(unary, image, w1=w1)
    unary.copy_(_inputs(torch, M, B=2, H=31, W=39, seed=9)[1])
    compat.mul_(0.7)
    g.replay()
    torch.cuda.synchronize()
    with torch.no_grad():
        want = nn.dense_crf(unary, None, compat_bi=compat[0], compat_sp=compat[1], features_bi=feats)
    assert float((out - want).abs().max()) <= BOUND


# ---- the feature range ----
@pytest.mark.parametrize("M", [21, 81])
def test_out_of_range_features_spoil_their_image_only(torch_cuda, M):
    torch = torch_cuda
    from dsrg_b200 import nn
    image, unary = _inputs(torch, M, B=3, H=29, W=35, seed=12)
    p = api.crf_params(1.0)
    feats = _features(torch, image, p)
    want = nn.dense_crf_inference(unary, None, features_bi=feats)
    bad = feats.clone()
    bad[1, 0, 3, 4] = 1000.0                       # pixels of image 1 far outside +-150
    bad[1, 2, 7, 9] = -1000.0
    got = nn.dense_crf_inference(unary, None, features_bi=bad)
    torch.cuda.synchronize()
    assert torch.isnan(got[1]).all()
    assert float((got[[0, 2]] - want[[0, 2]]).abs().max()) <= BOUND
    eng = nn.cached_engine(M, 29, 35, 0)
    assert eng.feature_range_flags(3).tolist() == [False, True, False]
    B, H, W = 3, 29, 35
    _, scores, _ = _post_inputs(torch, B, H, W, M, 2)
    peng = api.Engine(B, H, W, M)
    lab = torch.empty((B, H, W), dtype=torch.int32, device="cuda")
    probs = torch.empty((B, H, W, M), dtype=torch.float32, device="cuda")
    ok, ok_probs = torch.empty_like(lab), torch.empty_like(probs)
    peng.predict_mask_batch_learned_dev(scores, None, ok, p, features=feats, probs_out=ok_probs)
    peng.predict_mask_batch_learned_dev(scores, None, lab, p, features=bad, probs_out=probs)
    torch.cuda.synchronize()
    assert (lab[1] == -1).all() and torch.isnan(probs[1]).all()
    assert float((probs[[0, 2]] - ok_probs[[0, 2]]).abs().max()) <= BOUND
    sure = _sure(ok_probs[[0, 2]])
    assert torch.equal(lab[[0, 2]][sure], ok[[0, 2]][sure])
    assert peng.feature_range_flags(3).tolist() == [False, True, False]


# ---- refusals ----
def test_bad_arguments_are_refused_before_any_launch(torch_cuda):
    torch = torch_cuda
    from dsrg_b200 import nn, postprocess
    M = 6
    image, unary = _inputs(torch, M, B=2, H=17, W=19, seed=1)
    B, _, H, W = unary.shape
    eng = api.Engine(B, H, W, M)
    p = api.crf_params(1.0)
    feats = _features(torch, image, p)
    out = torch.empty_like(unary)
    L = _lib.lib()
    eng.take_launch_count()
    vp = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None   # noqa: E731
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    for img, f in ((image, feats), (None, None)):
        rc = L.dsrg_crf_batch_learned_dev(eng.h, vp(unary), B, api.LAYOUT_NCHW, vp(img), vp(f), C.byref(p), None,
                                          vp(out), api.LAYOUT_NCHW, s)
        assert rc == _lib.E_INVALID
    rc = L.dsrg_crf_batch_learned_dev(eng.h, vp(unary), B, 7, vp(image), None, C.byref(p), None, vp(out),
                                      api.LAYOUT_NCHW, s)
    assert rc == _lib.E_INVALID
    sc = [torch.zeros(B, M, 5, 5, device="cuda")]
    ptrs = (C.c_void_p * 1)(sc[0].data_ptr())
    hs, ws = (C.c_int * 1)(5), (C.c_int * 1)(5)
    lab = torch.empty((B, H, W), dtype=torch.int32, device="cuda")
    for img, f, mode, n in ((image, feats, 0, 1), (None, None, 0, 1), (image, None, 5, 1), (image, None, 1, 0)):
        rc = L.dsrg_predict_mask_batch_learned_dev(eng.h, ptrs, hs, ws, n, B, mode, vp(img), vp(f), 1e-5,
                                                   C.byref(p), None, None, vp(lab), None, s)
        assert rc == _lib.E_INVALID
    assert eng.take_launch_count() == 0
    with pytest.raises(ValueError):
        nn.dense_crf_inference(unary, image, features_bi=feats)
    with pytest.raises(ValueError):
        nn.dense_crf_inference(unary, None, features_bi=feats, theta_bi=torch.tensor([1.0] * 5))
    with pytest.raises(ValueError):
        nn.dense_crf_inference(unary, image, compat_bi=torch.zeros(M + 1, M + 1, device="cuda"))
    with pytest.raises(ValueError):
        nn.dense_crf_inference(unary, image, compat_bi=torch.zeros(M, M, device="cuda"), w1=_scalar(torch, 1.0))
    with pytest.raises(ValueError):
        nn.dense_crf_inference(unary, None, features_bi=feats[:, :4])
    with pytest.raises(ValueError):
        nn.dense_crf_inference(unary, image, theta_sp=torch.tensor([-1.0, 2.0]))
    with pytest.raises(ValueError):
        postprocess.predict_mask_batch_dev(image, sc, smooth=False, compat_bi=torch.zeros(M, M, device="cuda"))
    with pytest.raises(ValueError):
        postprocess.predict_mask_batch_dev(image, sc, features_bi=feats[:1])
    with pytest.raises(ValueError):
        postprocess.predict_masks_dev(list(image), sc, features_bi=[feats[0]])
