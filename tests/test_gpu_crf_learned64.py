"""The learned CRF at inference (Engine.crf_learned_dev, nn.dense_crf_inference, the learned predict_mask) against the
float64 restatements, per iteration, each image under its own bar (tests/crf_learned64_cases.py: LearnedTruth).

test_gpu_crf_learned.py checks the learned inference against the training forward and at the Potts identities; here
every case sits away from them (non-symmetric matrices, scaled and shifted features, both, one lattice's matrix zero,
other bandwidths) and is compared with the truth itself.  Cases: the three fused tile configurations at one label count
per padded width (4 to 32) in both unary and both output layouts, the hybrid-tile batch, gate 2 and both sides of the
blur switches, tiny shapes with 0..3 phantom lanes and the label-chunked path from 33 to 255 labels; the training
forward and backward with matrices at the widths the compat tests leave out (12, 16, 20 and 28); and the learned
predict_mask against post_oracle's steps with the float64 learned CRF in their CRF step.  Each case asserts the tile
path or blur branch it claims."""
import numpy as np
import pytest

import helpers
from crf_compat_cases import CompatTruth, compat_mats
from crf_grad_cases import grad_params, upstream
from crf_learned64_cases import (LEARNED_ITERS, LEARNED_M, LEARNED_TRAIN_M, LEARNED_WIDE_ITERS, LEARNED_WIDE_M,
                                 POST_B, POST_HYBRID_M, POST_HYBRID_SCORES, POST_KINDS, POST_M, POST_SEED, POST_SHAPE,
                                 POST_THETA_BI, POST_THETA_SP, POST_W1, POST_W2, LearnedTruth,
                                 kind_mats, kind_uses_features, learned_features, post_inputs, post_mats,
                                 post_oracle_case, post_params, predicted_paths, problem_for, reaches, sure,
                                 tag_ids)
from dsrg_b200 import api
from oracle import meanfield64

pytestmark = pytest.mark.gpu
ROWS = []          # (case, path, n_iters, device error, bar)
LAYOUTS = [(api.LAYOUT_NHWC, api.LAYOUT_NHWC), (api.LAYOUT_NCHW, api.LAYOUT_NCHW),
           (api.LAYOUT_NHWC, api.LAYOUT_NCHW), (api.LAYOUT_NCHW, api.LAYOUT_NHWC)]
HYBRID_ITERS = (0, 1, 2, 3)   # 321 x 321: the first three iterations, each through the hybrid tiles


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    if not ROWS:
        return
    print("\n%-44s %-10s %3s  %9s  %9s  %5s" % ("case", "path", "n", "dev err", "bar", "ratio"))
    worst = {}
    for case, path, n, err, bar in ROWS:
        print("%-44s %-10s %3d  %9.2e  %9.2e  %5.2f" % (case, path, n, err, bar, err / bar))
        worst[path] = max(worst.get(path, 0.0), err / bar)
    print("worst device error / bar per path: " + ", ".join("%s %.2f" % kv for kv in sorted(worst.items())))


def sm_count(torch):
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _nchw(torch, a):
    return torch.from_numpy(np.ascontiguousarray(np.transpose(a, (0, 3, 1, 2)))).cuda()


def _nhwc(t):
    return np.transpose(t.cpu().numpy(), (0, 2, 3, 1))


def check(case, path, got, truths, n):
    """got (B, H, W, M) device marginals after n iterations against the truths {b: LearnedTruth} of the compared
    images, each image against its own bar; the table keeps the image closest to its bar."""
    rows = {b: (float(np.abs(got[b] - t.q64[n]).max()), t.bar[n]) for b, t in truths.items()}
    b = max(rows, key=lambda k: rows[k][0] / rows[k][1])
    ROWS.append((case, path, n, rows[b][0], rows[b][1]))
    for b, (e, bar) in rows.items():
        assert e <= bar, (case, path, n, b, e, bar)


class Case(object):
    """One batch of a kind: the device inputs and the truths of the compared images.  problems caches each image's
    float64 lattices across label counts (key: image index and whether the kind uses features)."""

    def __init__(self, torch, kind, image, unary, params, compare, iters, seed, problems=None):
        B, H, W, M = unary.shape
        self.torch, self.kind, self.params, self.iters = torch, kind, params, iters
        self.unary = unary
        self.mus = kind_mats(kind, M, seed)
        problems = {} if problems is None else problems
        truths = {}
        for b in compare:
            key = (b, kind_uses_features(kind))
            if key not in problems:
                problems[key] = problem_for(kind, image[b], params)
            truths[b] = LearnedTruth(problems[key], unary[b], self.mus, iters)
        self.truths = truths
        self.d_image = torch.from_numpy(image).cuda()
        self.d_feats = None
        if kind_uses_features(kind):
            self.d_feats = _nchw(torch, np.stack([learned_features(image[b], params) for b in range(B)]))
        self.d_compat = None if self.mus is None else torch.from_numpy(np.stack(self.mus)).cuda()

    def device(self, eng, n, unary_layout=api.LAYOUT_NHWC, out_layout=api.LAYOUT_NHWC, B=None):
        """Engine.crf_learned_dev of the first B images after n iterations -> (B, H, W, M)."""
        torch = self.torch
        B = B or self.unary.shape[0]
        p = api.CrfParams.from_buffer_copy(self.params)
        p.n_iters = n
        un = self.unary[:B]
        u = torch.from_numpy(np.ascontiguousarray(un)).cuda() if unary_layout == api.LAYOUT_NHWC else _nchw(torch, un)
        out = torch.empty(un.shape if out_layout == api.LAYOUT_NHWC else (B, un.shape[3]) + un.shape[1:3],
                          device="cuda")
        eng.crf_learned_dev(u, None if self.d_feats is not None else self.d_image[:B], p, out,
                            features=None if self.d_feats is None else self.d_feats[:B].contiguous(),
                            compat=self.d_compat, unary_layout=unary_layout, out_layout=out_layout)
        torch.cuda.synchronize()
        return out.cpu().numpy() if out_layout == api.LAYOUT_NHWC else _nhwc(out)

    def run(self, eng, case, path, layouts=LAYOUTS, B=None):
        for n in self.iters:
            for ul, ol in layouts:
                name = case + ("" if (ul, ol) == LAYOUTS[0] else " %s>%s" % ("NCHW" if ul else "NHWC",
                                                                              "NCHW" if ol else "NHWC"))
                got = self.device(eng, n, ul, ol, B)
                check(name, path, got, {b: t for b, t in self.truths.items() if B is None or b < B}, n)


# ---- 1. the fused tile paths at every padded width ----
FUSED_KINDS = ("mats", "feats", "both")


@pytest.mark.parametrize("kind", FUSED_KINDS)
@pytest.mark.parametrize("path", sorted(helpers.MF64_PATH_CONFIG))
def test_fused_paths_every_width(torch_cuda, path, kind):
    img, sf = helpers.MF64_PATH_CONFIG[path]
    image = helpers.fused_images(img)
    B, H, W = image.shape[:3]
    params = helpers.mf64_problem_params(sf)
    assert reaches(predicted_paths(image, params, kind, sm_count(torch_cuda)), path), (path, kind)
    problems = {}
    for M in LEARNED_M:
        unary = helpers.log_unary(B, H, W, M, seed=200 + M)
        c = Case(torch_cuda, kind, image, unary, params, range(B), LEARNED_ITERS, M, problems)
        eng = api.Engine(B, H, W, M)
        c.run(eng, "%s %s M%d" % (path, kind, M), path)
        eng.close()


@pytest.mark.parametrize("kind", ["sp_only", "bi_only"])
def test_one_lattice_matrix(torch_cuda, kind):
    """One lattice's matrix zero: a failure names the lattice.  Both lattices on direct tiles somewhere, at the widths
    COMPAT_M leaves out."""
    for path in ("bi_direct", "sp_direct"):
        img, sf = helpers.MF64_PATH_CONFIG[path]
        image = helpers.fused_images(img)
        B, H, W = image.shape[:3]
        params = helpers.mf64_problem_params(sf)
        problems = {}
        for M in (9, 16, 18, 25):
            unary = helpers.log_unary(B, H, W, M, seed=300 + M)
            c = Case(torch_cuda, kind, image, unary, params, range(B), LEARNED_ITERS, M, problems)
            eng = api.Engine(B, H, W, M)
            c.run(eng, "%s %s M%d" % (path, kind, M), path, LAYOUTS[:2])
            eng.close()


def test_dense_crf_inference(torch_cuda):
    """nn.dense_crf_inference with matrices and features, at a width new to the matrix kernels (MP 20)."""
    torch = torch_cuda
    from dsrg_b200 import nn
    img, sf = helpers.MF64_PATH_CONFIG["bi_direct"]
    image = helpers.fused_images(img)
    B, H, W = image.shape[:3]
    M = 18
    params = helpers.mf64_problem_params(sf)
    c = Case(torch, "both", image, helpers.log_unary(B, H, W, M, seed=17), params, range(B), LEARNED_ITERS, 5)
    for n in LEARNED_ITERS:
        got = nn.dense_crf_inference(_nchw(torch, c.unary), None, scale_factor=sf, maxiter=n,
                                     compat_bi=c.d_compat[0], compat_sp=c.d_compat[1], features_bi=c.d_feats)
        torch.cuda.synchronize()
        check("dense_crf_inference both M%d" % M, "bi_direct", _nhwc(got), c.truths, n)


# ---- 2. the training forward and backward at the missing widths ----
def _train(torch, eng, images, unary, G, p, mus):
    B, M = unary.shape[0], unary.shape[-1]
    u, g, im = _nchw(torch, unary), _nchw(torch, G), torch.from_numpy(images).cuda()
    compat = torch.from_numpy(np.stack(mus)).cuda()
    q_hist = torch.empty((p.n_iters + 1,) + tuple(u.shape), device="cuda")
    gu, gm = torch.empty_like(u), torch.empty((B, 2, M, M), device="cuda")
    eng.crf_forward_train_compat_dev(u, im, p, compat, q_hist)
    eng.crf_backward_compat_dev(q_hist, im, p, compat, g, gu, grad_compat=gm)
    torch.cuda.synchronize()
    return _nhwc(q_hist[p.n_iters]), _nhwc(gu), gm.cpu().numpy()


def _train_case(torch, images, M, p, seed, compare, eng):
    B, H, W = images.shape[:3]
    unary = helpers.log_unary(B, H, W, M, seed, scale=1.0)
    G = np.stack([upstream(H, W, M, seed + b) for b in range(B)])
    mus = compat_mats("nonsym", M, seed)
    q, gu, gm = _train(torch, eng, images, unary, G, p, mus)
    for b in compare:
        CompatTruth(meanfield64.Problem(images[b], p), unary[b], G[b], p.n_iters, mus).check(
            q[b], gu[b], gm[b], "M%d image %d:" % (M, b))


@pytest.mark.parametrize("M", LEARNED_TRAIN_M)
def test_training_at_the_missing_widths(torch_cuda, M):
    img, sf = helpers.MF64_PATH_CONFIG["bi_direct"]
    images = helpers.fused_images(img)
    B, H, W = images.shape[:3]
    assert reaches(helpers.predict_tile_paths(images, sf, sm_count(torch_cuda)), "bi_direct")
    _train_case(torch_cuda, images, M, grad_params(sf, 3), 400 + M, range(B), api.Engine(B, H, W, M))


@pytest.mark.parametrize("M", LEARNED_TRAIN_M)
def test_training_at_the_missing_widths_hybrid(torch_cuda, M):
    images = helpers.hybrid_images()
    B, H, W = images.shape[:3]
    pred = helpers.predict_tile_paths(images, 1.0, sm_count(torch_cuda))
    b = int(np.argmax((pred["bi"] == "hybrid").sum(1)))
    eng = api.Engine(B, H, W, M)
    _train_case(torch_cuda, images, M, grad_params(1.0, 2), 500 + M, [b], eng)
    assert eng.hybrid_tiles == pred["hybrid_tiles"] > 0


# ---- 3. hybrid tiles ----
def test_hybrid_tiles(torch_cuda):
    torch = torch_cuda
    image = helpers.hybrid_images()
    B, H, W = image.shape[:3]
    params = helpers.mf64_problem_params(1.0)
    pred = helpers.predict_tile_paths(image, params, sm_count(torch))
    assert pred["hybrid_tiles"] > 0
    b = int(np.argmax((pred["bi"] == "hybrid").sum(1)))       # the image with the most hybrid tiles
    problems = {}
    for M in LEARNED_M:
        c = Case(torch, "mats", image, helpers.log_unary(B, H, W, M, seed=600 + M), params, [b], HYBRID_ITERS, M,
                 problems)
        eng = api.Engine(B, H, W, M)
        c.run(eng, "hybrid mats M%d (image %d)" % (M, b), "hybrid", LAYOUTS[:2])
        assert eng.hybrid_tiles == pred["hybrid_tiles"], M
        eng.close()
    for kind, M in (("feats", 9), ("both", 25)):
        c = Case(torch, kind, image, helpers.log_unary(B, H, W, M, seed=650 + M), params, [b], HYBRID_ITERS, M,
                 problems)
        eng = api.Engine(B, H, W, M)
        c.run(eng, "hybrid %s M%d (image %d)" % (kind, M, b), "hybrid", LAYOUTS[:2])
        assert eng.hybrid_tiles > 0, (kind, M)     # the features' lattice, not the image's: only that it is reached
        if kind == "both":
            # the same engine at B = 3 (too few tiles for the hybrid path), then at B = 5 again
            c3 = Case(torch, kind, image, c.unary, params, [min(b, 2)], (1, 3), M, problems)
            for n in c3.iters:
                check("direct %s M%d B=3" % (kind, M), "hybrid_off", c3.device(eng, n, B=3), c3.truths, n)
            assert eng.hybrid_tiles == 0
            c.run(eng, "hybrid %s M%d again" % (kind, M), "hybrid", LAYOUTS[:1])
            assert eng.hybrid_tiles > 0
        eng.close()


# ---- 4. gate 2 and the blur switches ----
def test_gate2_and_switches(torch_cuda):
    torch = torch_cuda
    image = helpers.seeded_images(*helpers.GATE2_SHAPE, ("noise", "noise"), helpers.GATE2_SEED)
    B, H, W = image.shape[:3]
    params = helpers.mf64_problem_params(1.0)
    problems = {}
    for M in helpers.MF64_GATE2_M:
        c = Case(torch, "mats", image, helpers.log_unary(B, H, W, M, seed=700 + M), params, [0], LEARNED_ITERS, M,
                 problems)
        eng = api.Engine(B, H, W, M)
        c.run(eng, "gate2 mats M%d" % M, "gate2", LAYOUTS[:2])
        assert helpers.blur_branch(H, W, eng.lattice_sizes(B)[1]) == "gate2"
        eng.close()
    for name, H, W, kinds, branch in helpers.SWITCH_CASES:
        image = helpers.seeded_images(H, W, kinds, helpers.GATE2_SEED)
        B = image.shape[0]
        c = Case(torch, "mats", image, helpers.log_unary(B, H, W, 21, seed=750 + H + W), params, [0], LEARNED_ITERS,
                 21)
        eng = api.Engine(B, H, W, 21)
        c.run(eng, "%s mats M21" % name, branch, LAYOUTS[:2])
        assert helpers.blur_branch(H, W, eng.lattice_sizes(B)[1]) == branch
        eng.close()


# ---- 5. tiny shapes: 0..3 phantom lanes in the last 4-pixel block ----
@pytest.mark.parametrize("kind", ["mats", "feats", "both"])
def test_tiny_shapes_phantom_lanes(torch_cuda, kind):
    M = helpers.MF64_TINY_M
    for H, W, img in helpers.MF64_TINY:
        image = np.stack([helpers.small_image(np.random.RandomState(helpers.MF64_TINY_SEED + b), H, W, img)
                          for b in range(2)])
        params = helpers.mf64_problem_params(1.0)
        c = Case(torch_cuda, kind, image, helpers.log_unary(2, H, W, M, seed=3), params, range(2), LEARNED_ITERS, 8)
        eng = api.Engine(2, H, W, M)
        c.run(eng, "tiny %dx%d %s" % (H, W, kind), "tiny")
        eng.close()


# ---- 6. the label-chunked path ----
@pytest.mark.parametrize("kind", ["mats", "feats", "both"])
@pytest.mark.parametrize("img", ["smooth", "noise"])
def test_wide_path(torch_cuda, img, kind):
    image = helpers.wide_images(img)
    B, H, W = image.shape[:3]
    params = helpers.mf64_problem_params(1.0)
    problems = {}
    for M in LEARNED_WIDE_M:
        c = Case(torch_cuda, kind, image, helpers.log_unary(B, H, W, M, seed=800 + M, scale=4.0), params, range(B),
                 LEARNED_WIDE_ITERS, M, problems)
        eng = api.Engine(B, H, W, M)
        c.run(eng, "wide %s %s M%d" % (img, kind, M), "wide", LAYOUTS[:2])
        eng.close()


# ---- 7. the learned predict_mask against the composed float64 oracle ----
POST_BOUND = 1e-4      # the post tests' bound on the marginals


def _sel(torch, tags):
    B, M = tags.shape
    present = torch.from_numpy(tags).cuda() > 0.5
    present[:, 0] = True
    ids = torch.arange(M, device="cuda", dtype=torch.int32).expand(B, M)
    order = torch.sort(torch.where(present, ids, ids + M), dim=1).values
    return torch.where(order < M, order, torch.full_like(order, -1)).contiguous()


def _device_kw(torch, kind, image, M):
    """(features, compat) device tensors of a predict_mask kind, either None, and its params."""
    p = post_params(kind)
    feats = None
    if kind in ("feats", "both"):
        feats = _nchw(torch, np.stack([learned_features(im, p) for im in image]))
    mus = post_mats(kind, M)
    return feats, None if mus is None else torch.from_numpy(np.stack(mus)).cuda(), p


def _postprocess_kw(torch, kind, feats, compat):
    """The learned keywords of postprocess.predict_mask_batch_dev for a kind."""
    if kind == "theta":
        scalar = lambda v: torch.tensor(v, device="cuda")   # noqa: E731
        return dict(theta_bi=torch.tensor(POST_THETA_BI), theta_sp=torch.tensor(POST_THETA_SP),
                    w1=scalar(POST_W1), w2=scalar(POST_W2))
    kw = {}
    if compat is not None:
        kw.update(compat_bi=compat[0], compat_sp=compat[1])
    if feats is not None:
        kw["features_bi"] = feats
    return kw


def _check_post(what, got_l, got_p, want_l, want_p, sel_ids=None):
    if got_p is not None:
        err = float(np.abs(got_p - want_p).max())
        ROWS.append((what, "predict_mask", 10, err, POST_BOUND))
        assert err <= POST_BOUND, (what, err)
    s = sure(want_p if sel_ids is None else want_p[..., sel_ids])
    assert s.mean() > 0.1, what                        # the comparison is not vacuous
    assert np.array_equal(got_l[s], want_l[s]), (what, int((got_l[s] != want_l[s]).sum()))


@pytest.mark.parametrize("mode", ["ms", "gt"])
@pytest.mark.parametrize("M", POST_M)
@pytest.mark.parametrize("kind", POST_KINDS)
def test_predict_mask_learned(torch_cuda, monkeypatch, kind, M, mode):
    """Engine.predict_mask_batch_learned_dev (labels and marginals) and postprocess.predict_mask_batch_dev (labels,
    through its keywords) against the composed oracle, every image of a B = 3 batch."""
    torch = torch_cuda
    from dsrg_b200 import postprocess
    B, (H, W) = POST_B, POST_SHAPE
    image, scores, tags = post_inputs(B, H, W, M, POST_SEED + M)
    if mode == "gt":
        scores = scores[:1]
    feats, compat, p = _device_kw(torch, kind, image, M)
    d_image = torch.from_numpy(image).cuda()
    d_scores = [torch.from_numpy(s).cuda() for s in scores]
    sel = _sel(torch, tags) if mode == "gt" else None
    eng = api.Engine(B, H, W, M)
    lab = torch.empty((B, H, W), dtype=torch.int32, device="cuda")
    probs = torch.empty((B, H, W, M), dtype=torch.float32, device="cuda")
    eng.predict_mask_batch_learned_dev(d_scores, None if feats is not None else d_image, lab, p,
                                       api.POST_SUM_SCORES if mode == "ms" else api.POST_ZOOM_PROBS,
                                       features=feats, compat=compat, sel=sel, probs_out=probs)
    pp = postprocess.predict_mask_batch_dev(d_image, d_scores, torch.from_numpy(tags).cuda() if mode == "gt" else None,
                                            mode=mode, **_postprocess_kw(torch, kind, feats, compat))
    torch.cuda.synchronize()
    lab, probs, pp = lab.cpu().numpy(), probs.cpu().numpy(), pp.cpu().numpy()
    for b in range(B):
        want_l, want_p = post_oracle_case(monkeypatch, kind, mode, image[b], [s[b] for s in scores], tags[b], M)
        sel_ids = None if mode == "ms" else [0] + tag_ids(tags[b])
        what = "%s %s M%d image %d" % (kind, mode, M, b)
        _check_post("engine " + what, lab[b], probs[b], want_l, want_p, sel_ids)
        _check_post("postprocess " + what, pp[b], None, want_l, want_p, sel_ids)


def test_predict_mask_learned_hybrid(torch_cuda, monkeypatch):
    """A batch large enough for hybrid tiles (B = 5 at 321 x 321, 41 x 41 scores), matrices and features."""
    torch = torch_cuda
    M = POST_HYBRID_M
    image = helpers.hybrid_images()
    B, H, W = image.shape[:3]
    rng = np.random.RandomState(POST_SEED)
    scores = [(rng.randn(B, M, *POST_HYBRID_SCORES) * 3).astype(np.float32)]
    pred = helpers.predict_tile_paths(image, 1.0, sm_count(torch))
    b = int(np.argmax((pred["bi"] == "hybrid").sum(1)))
    eng = api.Engine(B, H, W, M)
    for kind in ("mats", "both"):
        feats, compat, p = _device_kw(torch, kind, image, M)
        lab = torch.empty((B, H, W), dtype=torch.int32, device="cuda")
        probs = torch.empty((B, H, W, M), dtype=torch.float32, device="cuda")
        eng.predict_mask_batch_learned_dev([torch.from_numpy(scores[0]).cuda()],
                                           None if feats is not None else torch.from_numpy(image).cuda(), lab, p,
                                           api.POST_SUM_SCORES, features=feats, compat=compat, probs_out=probs)
        torch.cuda.synchronize()
        if kind == "mats":
            assert eng.hybrid_tiles == pred["hybrid_tiles"] > 0
        else:
            assert eng.hybrid_tiles > 0
        want_l, want_p = post_oracle_case(monkeypatch, kind, "ms", image[b], [scores[0][b]], None, M)
        _check_post("engine hybrid %s image %d" % (kind, b), lab[b].cpu().numpy(), probs[b].cpu().numpy(), want_l,
                    want_p)


def test_predict_masks_dev_mixed_sizes(torch_cuda, monkeypatch):
    """predict_masks_dev on mixed VOC sizes with per-image features and matrices: the groups keep each image's scores
    and features together.  Two images of different sizes are compared."""
    torch = torch_cuda
    from dsrg_b200 import postprocess
    M = 21
    rng = np.random.RandomState(POST_SEED + 1)
    sizes = [(375, 500), (500, 375), (375, 500), (333, 500)]
    ims = [helpers.small_image(rng, h, w, "photo") for h, w in sizes]
    sc = (rng.randn(len(ims), M, 41, 41) * 3).astype(np.float32)
    p = post_params("both")
    mus = post_mats("both", M)
    feats = [torch.from_numpy(np.ascontiguousarray(np.transpose(learned_features(im, p), (2, 0, 1)))).cuda()
             for im in ims]
    compat = torch.from_numpy(np.stack(mus)).cuda()
    got = postprocess.predict_masks_dev([torch.from_numpy(im).cuda() for im in ims], [torch.from_numpy(sc).cuda()],
                                        mode="ms", compat_bi=compat[0], compat_sp=compat[1], features_bi=feats)
    torch.cuda.synchronize()
    for i in (1, 3):
        want_l, want_p = post_oracle_case(monkeypatch, "both", "ms", ims[i], [sc[i]], None, M)
        _check_post("predict_masks_dev image %d %dx%d" % ((i,) + sizes[i]), got[i].cpu().numpy(), None, want_l,
                    want_p)
