"""GPU parity tests of the inference post-processing (SURVEY.md 8f rank 3) and of the re-shapeable engine
it runs on: dsrg_zoom_scores_*, dsrg_predict_mask_*, dsrg_engine_set_size against oracle/post_oracle.py
(the reference's predict_mask() tails restated with scipy + the CRF oracle)."""
import numpy as np
import pytest

from conftest import load_golden
from dsrg_b200 import api, pool, postprocess, synth
from helpers import make_golden
from oracle import crf_oracle, post_oracle

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


@pytest.mark.parametrize("h,w,H,W", [(41, 41, 120, 160), (31, 31, 97, 131), (51, 51, 60, 45), (41, 41, 41, 41),
                                     (41, 41, 20, 30), (7, 9, 1, 5), (41, 41, 375, 500)])
def test_zoom_scores_bit_exact(torch_cuda, h, w, H, W):
    from scipy import ndimage as nd
    rng = np.random.RandomState(h * 1000 + H)
    blob = (rng.randn(21, h, w) * 5).astype(np.float32)
    blob2 = (rng.randn(21, h + 3, w + 2) * 5).astype(np.float32)
    eng = pool.engine_for(H, W, 21)
    got = eng.zoom_scores_host(blob)
    want = nd.zoom(np.transpose(blob, [1, 2, 0]), (float(H) / h, float(W) / w, 1.0), order=1)
    assert got.shape == want.shape and np.array_equal(got, want)
    # scores_all += zoom(next scale)   (test-ms.py:97)
    eng.zoom_scores_host(blob2, out=got, accumulate=True)
    want = want + nd.zoom(np.transpose(blob2, [1, 2, 0]), (float(H) / (h + 3), float(W) / (w + 2), 1.0), order=1)
    assert np.array_equal(got, want)


def test_engine_set_size_reuses_buffers(torch_cuda):
    eng = api.Engine(1, 128, 160, 21)
    assert eng.capacity == (128, 160)
    for i, (H, W) in enumerate([(33, 45), (128, 160), (64, 50), (8, 160), (128, 7), (33, 45)]):
        eng.set_size(H, W)
        p = synth.make_problem(700 + i, H, W, image="smooth" if i % 2 == 0 else "noise")
        pr = np.transpose(p["probs"], (1, 2, 0)).copy()
        pr[pr < 1e-5] = 1e-5
        unary = np.log(pr)[None]
        got = eng.crf_host(unary, p["image"][None], api.crf_params(1.0))[0]
        want = crf_oracle.CRF(p["image"], unary[0], scale_factor=1.0)
        assert np.abs(got - want).max() <= TOL, (H, W)
    grown = eng.device_bytes   # staging is allocated once, by capacity
    eng.set_size(128, 160)
    eng.crf_host(np.zeros((1, 128, 160, 21), np.float32), np.zeros((1, 128, 160, 3), np.uint8), api.crf_params(1.0))
    assert eng.device_bytes == grown
    with pytest.raises(api.DsrgError):
        eng.set_size(129, 160)
    with pytest.raises(api.DsrgError):
        eng.set_size(0, 5)
    assert (eng.H, eng.W) == (128, 160)
    eng.close()


def test_engine_set_size_full_pass_bit_exact_srg(torch_cuda):
    """The training pass on a re-shaped engine: SRG seeds stay bit-exact, batch > 1."""
    from oracle import srg_oracle
    eng = api.Engine(3, 64, 64, 21)
    for (H, W) in [(41, 41), (64, 37), (23, 64)]:
        eng.set_size(H, W)
        b = synth.make_batch(3, H, W, cues="random", image="smooth", start=H)
        seeds = eng.srg_host(b["labels"], b["probs"], b["cues"], 0.99, 0.85)
        for i in range(3):
            want = srg_oracle.srg_closed_form(b["labels"][i], b["cues"][i], b["probs"][i], 0.99, 0.85)
            assert np.array_equal(seeds[i], want)
    eng.close()


@pytest.mark.parametrize("H,W,sizes,index", [(120, 160, (31, 41, 51), 0), (97, 75, (41,), 1), (150, 200, (21, 31), 2)])
def test_predict_mask_ms(torch_cuda, H, W, sizes, index):
    s = synth.make_score_blobs(index, H, W, sizes)
    want_lab, want_p = post_oracle.predict_mask_ms(s["image"], s["blobs"], smooth=True)
    got_lab, got_p = postprocess.predict_mask_ms(s["image"], s["blobs"], smooth=True, return_probs=True)
    assert got_lab.shape == (H, W) and got_lab.dtype == np.int64
    assert np.abs(got_p - want_p).max() <= TOL
    flips = labels_agree(got_lab, want_lab, want_p)
    assert flips <= 1e-3 * H * W
    assert len(np.unique(want_lab)) >= 2          # the case is not degenerate
    # smooth=False: soft-max only
    want_lab, want_p = post_oracle.predict_mask_ms(s["image"], s["blobs"], smooth=False)
    got_lab, got_p = postprocess.predict_mask_ms(s["image"], s["blobs"], smooth=False, return_probs=True)
    np.testing.assert_allclose(got_p, want_p, rtol=2e-6, atol=1e-9)
    labels_agree(got_lab, want_lab, want_p, margin=1e-6)
    assert np.array_equal(postprocess.predict_mask_ms(s["image"], s["blobs"], smooth=False), got_lab)


@pytest.mark.parametrize("H,W,size,index", [(120, 160, 41, 3), (64, 90, 33, 4)])
def test_predict_mask_gt(torch_cuda, H, W, size, index):
    s = synth.make_score_blobs(index, H, W, (size,))
    for smooth in (True, False):
        want_lab, want_p = post_oracle.predict_mask_gt(s["image"], s["blobs"][0], s["tags"], smooth=smooth)
        got_lab, got_p = postprocess.predict_mask_gt(s["image"], s["blobs"][0], s["tags"], smooth=smooth,
                                                     return_probs=True)
        sel = [0] + s["tags"].tolist()
        assert set(np.unique(got_lab)) <= set(sel)
        if smooth:
            assert np.abs(got_p - want_p).max() <= TOL
            labels_agree(got_lab, want_lab, want_p, sel)
        else:
            np.testing.assert_allclose(got_p, want_p, rtol=4e-6, atol=1e-9)
            labels_agree(got_lab, want_lab, want_p, sel, margin=1e-6)


def test_predict_mask_voc_size_and_dev_entry(torch_cuda):
    """A VOC-sized image (375x500) through the host entry point, and the same through the *_dev one."""
    import torch
    H, W = 375, 500
    s = synth.make_score_blobs(9, H, W, (31, 41, 51))
    want_lab, want_p = post_oracle.predict_mask_ms(s["image"], s["blobs"], smooth=True)
    got_lab, got_p = postprocess.predict_mask_ms(s["image"], s["blobs"], smooth=True, return_probs=True)
    assert np.abs(got_p - want_p).max() <= TOL
    assert labels_agree(got_lab, want_lab, want_p) <= 1e-3 * H * W
    eng = pool.engine_for(H, W, 21)
    blobs = [torch.from_numpy(b).cuda() for b in s["blobs"]]
    im = torch.from_numpy(s["image"]).cuda()
    res = torch.empty((H, W), dtype=torch.int32, device="cuda")
    pr = torch.empty((H, W, 21), dtype=torch.float32, device="cuda")
    eng.predict_mask_dev(blobs, im, res, probs_out=pr)
    torch.cuda.synchronize()
    assert np.abs(pr.cpu().numpy() - want_p).max() <= TOL
    labels_agree(res.cpu().numpy(), want_lab, want_p)


@pytest.mark.parametrize("case", make_golden.POST_CASES, ids=[c[0] for c in make_golden.POST_CASES])
def test_predict_mask_against_frozen_golden(torch_cuda, case):
    name, mode, H, W, sizes, index = case
    g = load_golden("post_oracle_%s.npz" % name)
    im, blobs, tags = make_golden.post_inputs(H, W, sizes, index)
    if mode == "ms":
        lab, probs = postprocess.predict_mask_ms(im, blobs, return_probs=True)
        sel = None
    else:
        lab, probs = postprocess.predict_mask_gt(im, blobs[0], tags, return_probs=True)
        sel = [0] + list(tags)
    assert np.abs(probs - g["probs"]).max() <= TOL
    labels_agree(lab, g["labels"], g["probs"], sel)


def test_predict_mask_argument_errors(torch_cuda):
    eng = pool.engine_for(40, 40, 21)
    blob = np.zeros((21, 10, 10), np.float32)
    im = np.zeros((40, 40, 3), np.uint8)
    with pytest.raises(api.DsrgError):
        eng.predict_mask_host([blob], im, mode=7)
    with pytest.raises(api.DsrgError):
        eng.predict_mask_host([blob, blob], im, mode=api.POST_ZOOM_PROBS)
    with pytest.raises(api.DsrgError):
        eng.predict_mask_host([blob], im, labels_sel=[0, 21])
    with pytest.raises(api.DsrgError):
        eng.predict_mask_host([blob], None, smooth=True)
    # at most 16 score maps, in both entry points, refused before any launch
    torch = torch_cuda
    d_blob, d_im = torch.from_numpy(blob).cuda(), torch.from_numpy(im).cuda()
    res = torch.empty((40, 40), dtype=torch.int32, device="cuda")
    eng.take_launch_count()
    with pytest.raises(api.DsrgError):
        eng.predict_mask_host([blob] * 17, im)
    with pytest.raises(api.DsrgError):
        eng.predict_mask_dev([d_blob] * 17, d_im, res)
    assert eng.take_launch_count() == 0
    assert eng.predict_mask_host([blob], None, smooth=False).shape == (40, 40)


def test_crf_function_many_sizes_one_engine(torch_cuda):
    """krahenbuhl2013.CRF over images of changing size (grow, shrink, transpose) -- one pooled engine."""
    import fake_caffe
    fake_caffe.install()
    import krahenbuhl2013
    pool.clear()
    for i, (H, W) in enumerate([(40, 60), (60, 40), (90, 130), (33, 45), (130, 90)]):
        p = synth.make_problem(800 + i, H, W, image="smooth")
        pr = np.transpose(p["probs"], (1, 2, 0)).copy()
        pr[pr < 1e-5] = 1e-5
        got = krahenbuhl2013.CRF(p["image"], np.log(pr), scale_factor=1.0)
        want = crf_oracle.CRF(p["image"], np.log(pr), scale_factor=1.0)
        assert np.abs(got - want).max() <= TOL
    assert len(pool._ENGINES) == 1


def test_per_image_callers_replay_graphs_across_sizes(torch_cuda):
    """The evaluation tools meet the same image sizes again and again: the post-processing of one image and a
    DenseCRF object's inference are replayed as CUDA graphs per size (post.cu:predict_mask_batch, api.cu:densecrf_run),
    also when another size ran on the shared engine in between (the replayed graph then contains the rebuild of
    the shared spatial lattice).  Results equal the plain launches up to the float atomics' noise."""
    import fake_caffe
    fake_caffe.install()
    import krahenbuhl2013
    pool.clear()
    cases = [synth.make_score_blobs(40 + i, H, W, (31, 41)) for i, (H, W) in enumerate([(90, 120), (120, 90), (75, 100)])]
    crf_cases = []
    for i, (H, W) in enumerate([(60, 80), (80, 60)]):
        p = synth.make_problem(900 + i, H, W, image="smooth")
        pr = np.transpose(p["probs"], (1, 2, 0)).copy()
        pr[pr < 1e-5] = 1e-5
        crf_cases.append((p["image"], np.log(pr)))
    eng = pool.engine_for(120, 120, 21)
    eng.set_graphs(False)
    want = [postprocess.predict_mask_ms(c["image"], c["blobs"], return_probs=True) for c in cases]
    want_crf = [krahenbuhl2013.CRF(im, u, scale_factor=1.0) for im, u in crf_cases]
    eng.set_graphs(True)
    r0 = eng.graph_replays
    for rnd in range(4):
        for c, (wl, wp) in zip(cases, want):
            lab, pr = postprocess.predict_mask_ms(c["image"], c["blobs"], return_probs=True)
            assert np.abs(pr - wp).max() <= TOL
            labels_agree(lab, wl, wp)
        for (im, u), w in zip(crf_cases, want_crf):
            assert np.abs(krahenbuhl2013.CRF(im, u, scale_factor=1.0) - w).max() <= TOL
    assert eng is pool.engine_for(120, 120, 21)          # still the one pooled engine
    assert eng.graph_replays - r0 >= 2 * (len(cases) + len(crf_cases))   # rounds 3 and 4 are replays
