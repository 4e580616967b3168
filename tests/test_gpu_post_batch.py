"""GPU tests of the batched inference post-processing (dsrg_predict_mask_batch_*, postprocess.predict_masks_* and
predict_mask_batch_dev): without the CRF every image of a batch is bit-identical to the per-image pass on that image
alone; with it the marginals follow the CRF's 1e-4 bound against oracle/post_oracle.py and the per-image pass."""
import ctypes as C

import numpy as np
import pytest

from dsrg_b200 import _lib, api, pool, postprocess, synth
from oracle import post_oracle

pytestmark = pytest.mark.gpu

TOL = 1e-4   # CRF marginals, as everywhere else (DESIGN.md section 3)


def labels_agree(got, want_labels, want_probs, sel=None, margin=4 * TOL):
    """Label maps must be equal except where the oracle's own decision is a near-tie (top-2 margin
    within the CRF parity bound); returns the number of such pixels."""
    bad = got != want_labels
    if not bad.any():
        return 0
    p = want_probs if sel is None else want_probs[:, :, sel]
    top2 = np.sort(p, axis=2)[:, :, -2:]
    gap = top2[:, :, 1] - top2[:, :, 0]
    assert (gap[bad] <= margin).all(), "label differs where the oracle's margin is %g" % gap[bad].max()
    return int(bad.sum())


def score_shapes(H, W, spec):
    """("abs", sizes): the square maps of test-ms.py's absolute input sizes; ("rel", factors): the maps of
    test-ms-f.py's zoom factors, which follow the image's aspect (stride 8 of the network input)."""
    kind, vals = spec
    if kind == "abs":
        return [(v, v) for v in vals]
    return [((int(round(H * f)) + 7) // 8, (int(round(W * f)) + 7) // 8) for f in vals]


def sel_rows(B, M, rng):
    """Rows that cover every selection kind: unsorted, duplicate ids, [0] only, every label without a -1 (in a
    shuffled order), and a short ascending tag list."""
    rows = np.full((B, M), -1, np.int32)
    for b in range(B):
        kind = b % 5
        if kind == 0:
            r = [0, 7 % M, 3 % M, 12 % M]
        elif kind == 1:
            r = [0, 5 % M, 5 % M, 2 % M, 0]
        elif kind == 2:
            r = [0]
        elif kind == 3:
            r = list(rng.permutation(M))
        else:
            r = [0] + sorted(rng.choice(np.arange(1, M), size=min(3, M - 1), replace=False).tolist())
        rows[b, :len(r)] = r
    return rows


def row_list(row):
    r = row.tolist()
    return r[:r.index(-1)] if -1 in r else r


BITEXACT = [  # mode, M, score spec, B, H, W
    ("ms", 21, ("abs", (41, 31, 51)), 16, 375, 500),
    ("ms", 21, ("rel", (0.75, 1.25)), 5, 97, 131),
    ("ms", 21, ("abs", (41,)), 1, 375, 500),
    ("ms", 81, ("rel", (1.0, 0.5, 1.5)), 2, 375, 500),
    ("ms", 81, ("abs", (33, 21)), 5, 61, 83),
    ("gt", 21, ("abs", (41,)), 5, 375, 500),
    ("gt", 21, ("rel", (1.0,)), 16, 61, 83),
    ("gt", 81, ("rel", (0.5,)), 2, 97, 131),
    ("gt", 81, ("abs", (41,)), 1, 375, 500),
]


@pytest.mark.parametrize("mode,M,spec,B,H,W", BITEXACT,
                         ids=["%s-M%d-%s%d-B%d-%dx%d" % (c[0], c[1], c[2][0], len(c[2][1]), c[3], c[4], c[5])
                              for c in BITEXACT])
def test_batch_equals_per_image_bit_exact(torch_cuda, mode, M, spec, B, H, W):
    torch = torch_cuda
    rng = np.random.RandomState(B * 1000 + H + M)
    shapes = score_shapes(H, W, spec)
    scores = [torch.from_numpy((rng.randn(B, M, h, w) * 3).astype(np.float32)).cuda() for h, w in shapes]
    images = torch.from_numpy(rng.randint(0, 256, (B, H, W, 3)).astype(np.uint8)).cuda()
    pmode = _lib.POST_SUM_SCORES if mode == "ms" else _lib.POST_ZOOM_PROBS
    params = api.crf_params(1.0)
    rows = torch.from_numpy(sel_rows(B, M, rng)).cuda()
    eng = pool.batch_engine_for(B, H, W, M)
    one = pool.engine_for(H, W, M)
    for sel in (None, rows):
        res = torch.full((B, H, W), -7, dtype=torch.int32, device="cuda")
        prb = torch.full((B, H, W, M), float("nan"), device="cuda")
        eng.predict_mask_batch_dev(scores, images, res, params, pmode, postprocess.EPS, False, sel, prb)
        for b in range(B):
            r1 = torch.empty((H, W), dtype=torch.int32, device="cuda")
            p1 = torch.empty((H, W, M), device="cuda")
            lsel = None if sel is None else row_list(sel[b].cpu().numpy())
            one.predict_mask_dev([s[b] for s in scores], images[b], r1, params, pmode, postprocess.EPS, False, lsel,
                                 p1)
            assert torch.equal(res[b], r1), (b, lsel)
            assert torch.equal(prb[b], p1), b
    # the host entry point computes the same
    got, got_p = eng.predict_mask_batch_host([s.cpu().numpy() for s in scores], None, params, pmode, postprocess.EPS,
                                             False, rows.cpu().numpy(), True)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(got, res.cpu().numpy())
    np.testing.assert_array_equal(got_p, prb.cpu().numpy())


def _crf_case(B, H, W, M, sizes, image, start):
    cases = [synth.make_score_blobs(start + i, H, W, sizes, C=M, image=image) for i in range(B)]
    ims = np.stack([c["image"] for c in cases])
    blobs = [np.stack([c["blobs"][k] for c in cases]) for k in range(len(sizes))]
    return cases, ims, blobs


@pytest.mark.parametrize("mode,M,B,H,W,sizes,image", [
    ("ms", 21, 5, 375, 500, (31, 41, 51), "photo"),     # 5 x 752 tiles, >= 16 per SM: the pass takes hybrid tiles
    ("gt", 21, 5, 97, 131, (41,), "smooth"),
    ("ms", 81, 2, 61, 83, (21, 33), "smooth"),
])
def test_batch_crf_against_oracle_and_per_image(torch_cuda, mode, M, B, H, W, sizes, image):
    cases, ims, blobs = _crf_case(B, H, W, M, sizes, image, 60 + B)
    eng = pool.batch_engine_for(B, H, W, M)
    pmode = _lib.POST_SUM_SCORES if mode == "ms" else _lib.POST_ZOOM_PROBS
    sel = None
    if mode == "gt":
        sel = np.full((B, M), -1, np.int32)
        for b, c in enumerate(cases):
            r = [0] + c["tags"].tolist()
            sel[b, :len(r)] = r
    lab, probs = eng.predict_mask_batch_host(blobs, ims, api.crf_params(1.0), pmode, postprocess.EPS, True, sel, True)
    if image == "photo":
        assert eng.hybrid_tiles > 0
    flips = 0
    for b, c in enumerate(cases):
        if mode == "ms":
            want_lab, want_p = post_oracle.predict_mask_ms(c["image"], [x[b] for x in blobs], smooth=True)
            one_lab, one_p = postprocess.predict_mask_ms(c["image"], [x[b] for x in blobs], return_probs=True)
            s = None
        else:
            want_lab, want_p = post_oracle.predict_mask_gt(c["image"], blobs[0][b], c["tags"], smooth=True)
            one_lab, one_p = postprocess.predict_mask_gt(c["image"], blobs[0][b], c["tags"], return_probs=True)
            s = [0] + c["tags"].tolist()
        assert np.abs(probs[b] - want_p).max() <= TOL, b
        assert np.abs(probs[b] - one_p).max() <= TOL, b
        flips += labels_agree(lab[b], want_lab, want_p, s)
        labels_agree(lab[b], one_lab, one_p, s)
    assert flips <= 1e-3 * B * H * W


def _mixed_list(n, M=21, seed=5):
    rng = np.random.RandomState(seed)
    kinds = [(97, 131, (31, 41)), (131, 97, (41, 21)), (64, 90, (33, 41)), (97, 131, (41, 31))]
    ims, scores, tags = [], [], []
    for i in range(n):
        H, W, sizes = kinds[rng.randint(len(kinds))]
        c = synth.make_score_blobs(200 + i, H, W, sizes, C=M)
        ims.append(c["image"])
        scores.append(c["blobs"])
        tags.append(rng.permutation(c["tags"]))   # the caller's order decides exact ties
    return ims, scores, tags


def test_host_grouping_in_input_order(torch_cuda):
    ims, scores, tags = _mixed_list(11)
    for smooth in (False, True):
        got, got_p = postprocess.predict_masks_ms(ims, scores, smooth=smooth, batch=4, return_probs=True)
        got_gt = postprocess.predict_masks_gt(ims, [s[0] for s in scores], tags, smooth=smooth, batch=3)
        assert len(got) == len(got_gt) == len(ims)
        for i, im in enumerate(ims):
            lab, p = postprocess.predict_mask_ms(im, scores[i], smooth=smooth, return_probs=True)
            lab_gt, p_gt = postprocess.predict_mask_gt(im, scores[i][0], tags[i], smooth=smooth, return_probs=True)
            assert got[i].dtype == np.int64 and got[i].shape == im.shape[:2]
            assert got_gt[i].dtype == np.int64 and got_gt[i].shape == im.shape[:2]
            if not smooth:
                np.testing.assert_array_equal(got[i], lab)
                np.testing.assert_array_equal(got_p[i], p)
                np.testing.assert_array_equal(got_gt[i], lab_gt)
            else:
                assert np.abs(got_p[i] - p).max() <= TOL
                labels_agree(got[i], lab, p)
                labels_agree(got_gt[i], lab_gt, p_gt, [0] + tags[i].tolist())


def _dev_inputs(torch, B=3, H=97, W=131, M=21, seed=8):
    rng = np.random.RandomState(seed)
    cases = [synth.make_score_blobs(300 + seed * 10 + i, H, W, (41,), C=M) for i in range(B)]
    images = torch.from_numpy(np.stack([c["image"] for c in cases])).cuda()
    scores = [torch.from_numpy(np.stack([c["blobs"][0] for c in cases])).cuda()]
    tags = np.zeros((B, 1, 1, M), np.float32)
    for b, c in enumerate(cases):
        tags[b, 0, 0, c["tags"]] = 1
    tags[:, 0, 0, rng.randint(1, M)] = 1
    return cases, images, scores, torch.from_numpy(tags).cuda()


def test_dev_path_side_stream_matches_host(torch_cuda):
    torch = torch_cuda
    cases, images, scores, tags = _dev_inputs(torch)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ms = postprocess.predict_mask_batch_dev(images, scores, mode="ms", smooth=False)
        gt = postprocess.predict_mask_batch_dev(images, scores, labels=tags, mode="gt", smooth=False)
        gt_s = postprocess.predict_mask_batch_dev(images, scores, labels=tags, mode="gt", smooth=True)
    side.synchronize()
    assert ms.dtype == torch.int32 and tuple(ms.shape) == tuple(images.shape[:3])
    blobs = scores[0].cpu().numpy()
    for b, c in enumerate(cases):
        tag_ids = np.where(tags[b, 0, 0].cpu().numpy() > 0.5)[0]
        tag_ids = tag_ids[tag_ids > 0]
        np.testing.assert_array_equal(ms[b].cpu().numpy(), postprocess.predict_mask_ms(c["image"], [blobs[b]],
                                                                                        smooth=False))
        np.testing.assert_array_equal(gt[b].cpu().numpy(), postprocess.predict_mask_gt(c["image"], blobs[b], tag_ids,
                                                                                        smooth=False))
        lab, p = postprocess.predict_mask_gt(c["image"], blobs[b], tag_ids, return_probs=True)
        labels_agree(gt_s[b].cpu().numpy(), lab, p, [0] + tag_ids.tolist())
    # the confusion matrix counts the device result as it stands
    gt_maps = torch.from_numpy(np.stack([c["image"][:, :, 0] % 21 for c in cases]).astype(np.uint8)).cuda()
    conf = api.Confusion(21)
    conf.add_dev(gt_maps, gt)
    m, inv = conf.read()
    conf.close()
    assert int(m.sum()) == gt.numel() and int(inv.sum()) == 0


def test_dev_path_in_a_cuda_graph_follows_the_tags(torch_cuda):
    torch = torch_cuda
    cases, images, scores, tags = _dev_inputs(torch, seed=9)
    tags_a = tags.clone()
    tags_b = torch.zeros_like(tags)
    tags_b[:, 0, 0, 0] = 1
    tags_b[:, 0, 0, 1:4] = 1
    for smooth in (False, True):
        tags.copy_(tags_a)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):   # warm-up: the engine, its staging, torch's kernels
            for _ in range(2):
                postprocess.predict_mask_batch_dev(images, scores, labels=tags, mode="gt", smooth=smooth)
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            res = postprocess.predict_mask_batch_dev(images, scores, labels=tags, mode="gt", smooth=smooth)
        for t in (tags_a, tags_b, tags_a):
            tags.copy_(t)
            graph.replay()
            want = postprocess.predict_mask_batch_dev(images, scores, labels=tags, mode="gt", smooth=smooth)
            torch.cuda.synchronize()
            if not smooth:
                assert torch.equal(res, want)
            else:
                assert float((res == want).float().mean()) >= 0.999
            allowed = {0} | set(torch.nonzero(t[0, 0, 0] > 0.5).flatten().tolist())
            assert set(torch.unique(res[0]).tolist()) <= allowed
        del graph


def test_repeated_eager_call_replays_the_engine_graph(torch_cuda):
    torch = torch_cuda
    cases, images, scores, tags = _dev_inputs(torch, seed=10)
    out = torch.empty(tuple(images.shape[:3]), dtype=torch.int32, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        first = postprocess.predict_mask_batch_dev(images, scores, mode="ms", out=out).clone()
        eng = pool.batch_engine_for(*images.shape[:3], 21)
        r0 = eng.graph_replays
        for _ in range(3):
            postprocess.predict_mask_batch_dev(images, scores, mode="ms", out=out)
    side.synchronize()
    assert eng.graph_replays > r0
    assert float((out == first).float().mean()) >= 0.999


def test_errors_before_any_launch(torch_cuda):
    torch = torch_cuda
    L = _lib.lib()
    B, H, W, M, h = 3, 40, 48, 21, 12
    eng = api.Engine(B, H, W, M)
    rng = np.random.RandomState(3)
    dsc = torch.from_numpy(rng.randn(B, M, h, h).astype(np.float32)).cuda()
    hsc = dsc.cpu().numpy()
    dimg = torch.zeros((B, H, W, 3), dtype=torch.uint8, device="cuda")
    himg = np.zeros((B, H, W, 3), np.uint8)
    dres = torch.empty((B, H, W), dtype=torch.int32, device="cuda")
    hres = np.empty((B, H, W), np.int32)
    prm = C.byref(api.crf_params(1.0))
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def ptrs(p, n):
        return (C.c_void_p * max(n, 1))(*([p] * n))

    def ints(v, n):
        return (C.c_int * max(n, 1))(*([v] * n))

    def dev(n=1, b=B, mode=0, hh=h, ww=h, img=True, res=True, sc=True, smooth=1, sel=None):
        return L.dsrg_predict_mask_batch_dev(C.c_void_p(eng.h), ptrs(dsc.data_ptr(), n) if sc else None, ints(hh, n),
                                             ints(ww, n), n, b, mode, C.c_void_p(dimg.data_ptr()) if img else None,
                                             1e-5, smooth, prm, sel, C.c_void_p(dres.data_ptr()) if res else None,
                                             None, s)

    def host(n=1, b=B, mode=0, hh=h, ww=h, img=True, res=True, sc=True, smooth=1, sel=None):
        return L.dsrg_predict_mask_batch_host(C.c_void_p(eng.h), ptrs(hsc.ctypes.data, n) if sc else None,
                                              ints(hh, n), ints(ww, n), n, b, mode,
                                              C.c_void_p(himg.ctypes.data) if img else None, 1e-5, smooth, prm,
                                              None if sel is None else C.c_void_p(sel.ctypes.data),
                                              C.c_void_p(hres.ctypes.data) if res else None, None)

    bad_sel = np.full((B, M), -1, np.int32)
    bad_sel[:, 0] = 0
    bad_sel[1, 1] = M
    cases = [dict(b=0), dict(b=B + 1), dict(n=0), dict(n=17), dict(mode=1, n=2), dict(mode=5),
             dict(hh=H * W), dict(hh=0), dict(img=False), dict(res=False), dict(sc=False)]
    dev_id = torch.cuda.current_device()
    eng.take_launch_count()
    for kw in cases:
        for f in (dev, host):
            assert f(**kw) == _lib.E_INVALID, (f.__name__, kw)
            assert eng.take_launch_count() == 0, (f.__name__, kw)
            assert torch.cuda.current_device() == dev_id
    assert host(sel=bad_sel) == _lib.E_INVALID
    assert "image 1: selected label 21 outside [0, 21)" in L.dsrg_last_error().decode()
    assert eng.take_launch_count() == 0
    # without the CRF the image may be NULL
    assert host(img=False, smooth=0) == _lib.OK
    # _dev reports a bad row in that image's result: every pixel -1, the others untouched by it
    dsel = torch.from_numpy(bad_sel).cuda()
    assert dev(sel=C.c_void_p(dsel.data_ptr())) == _lib.OK
    torch.cuda.synchronize()
    r = dres.cpu().numpy()
    assert (r[1] == -1).all() and (r[0] == 0).all() and (r[2] == 0).all()
    eng.close()
    # the Python device path refuses before it queues anything
    with pytest.raises(ValueError):
        postprocess.predict_mask_batch_dev(dimg, [dsc], mode="gt", labels=torch.zeros((B, M + 1), device="cuda"))
    with pytest.raises(ValueError):
        postprocess.predict_mask_batch_dev(dimg, [dsc, dsc], mode="gt")
    with pytest.raises(ValueError):
        postprocess.predict_mask_batch_dev(dimg, [dsc[:2]], mode="ms")
    with pytest.raises(ValueError):
        postprocess.predict_mask_batch_dev(dimg, [dsc.double()], mode="ms")
    with pytest.raises(ValueError):
        postprocess.predict_mask_batch_dev(dimg, [dsc], mode="xx")
