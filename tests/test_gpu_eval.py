"""GPU tests of segmentation scoring (csrc/eval.cu, dsrg_confusion_*, dsrg_b200/metrics.py) and of the predict_mask
post-processing at COCO's 81 labels (csrc/post.cu's wide soft-max).  The device matrix must equal an int64 numpy
bincount restatement bit for bit; the drop-in classes must equal the reference's frozen outputs
(tests/golden/eval_ref.npz)."""
import warnings

import numpy as np
import pytest

from conftest import load_golden
from dsrg_b200 import api, metrics, pool, postprocess, synth
from oracle import post_oracle

pytestmark = pytest.mark.gpu

TOL = 1e-4


def want_matrix(gt, pred, K):
    """generateM's rules restated with an int64 bincount: bin iff gt < K and 0 <= pred < K."""
    gt, pred = np.asarray(gt).reshape(-1).astype(np.int64), np.asarray(pred).reshape(-1).astype(np.int64)
    pv = (pred >= 0) & (pred < K)
    ok = (gt < K) & pv
    M = np.bincount(gt[ok] * K + pred[ok], minlength=K * K).reshape(K, K).astype(np.uint64)
    inv = np.array([((gt >= K) & (gt != 255)).sum(), ((gt < K) & ~pv).sum()], np.uint64)
    return M, inv


def labels(rng, n, K, dtype):
    """Mostly background, runs of one label, 255 and gt >= K pixels, predictions >= K and (int32) negative."""
    gt = np.zeros(n, np.int64)
    if n:
        cuts = np.sort(rng.randint(0, n, max(1, n // 5000)))
        gt = np.repeat(rng.randint(0, K, cuts.size + 1), np.diff(np.r_[0, cuts, n]))
        gt[rng.rand(n) < 0.4] = 0
        gt[rng.rand(n) < 0.05] = 255
        gt[rng.rand(n) < 0.01] = rng.randint(min(K, 254), 255)
    pred = np.where(rng.rand(n) < 0.7, np.minimum(gt, K - 1), rng.randint(0, K, n))
    bad = rng.rand(n) < 0.01
    pred[bad] = rng.randint(K, 256, int(bad.sum())) if dtype == np.uint8 else rng.randint(-300, 300, int(bad.sum()))
    if dtype == np.uint8:
        pred = np.clip(pred, 0, 255)
    return gt.astype(np.uint8), pred.astype(dtype)


def dev_at(torch, a, offset):
    """a copy of `a` on the device starting `offset` bytes after a 256-byte aligned allocation"""
    buf = torch.zeros(a.nbytes + offset + 64, dtype=torch.uint8, device="cuda")
    view = buf[offset:offset + a.nbytes]
    view.copy_(torch.from_numpy(a.view(np.uint8).copy()))
    return view if a.dtype == np.uint8 else view.view(torch.int32)


@pytest.mark.parametrize("K", [2, 21, 22, 81, 82, 200, 255])
@pytest.mark.parametrize("dtype", [np.uint8, np.int32], ids=["u8", "i32"])
def test_device_matrix_bit_exact(torch_cuda, K, dtype):
    torch = torch_cuda
    rng = np.random.RandomState(K * 7 + (dtype == np.int32))
    conf = api.Confusion(K)
    acc_M, acc_inv = np.zeros((K, K), np.uint64), np.zeros(2, np.uint64)
    sizes = [0, 1, 15, 17, 4097, 3_000_017]
    for j, n in enumerate(sizes):
        gt, pred = labels(rng, n, K, dtype)
        go = (3 * j + 1) % 16                                  # gt offset 1..15
        # pred offset: the same as gt's or another one, so both the 16-byte and the element-wise pred loads run
        po = (go if j % 2 else 7 * j % 16) if dtype == np.uint8 else 4 * ((j + 1) % 4)
        conf.add_dev(dev_at(torch, gt, go), dev_at(torch, pred, po))
        M, inv = want_matrix(gt, pred, K)
        acc_M += M
        acc_inv += inv
        one = api.Confusion(K)
        one.add_dev(dev_at(torch, gt, go), dev_at(torch, pred, po))
        got_M, got_inv = one.read()
        assert np.array_equal(got_M, M) and np.array_equal(got_inv, inv), (n, go, po)
        one.reset()
        one.add_host(gt, pred)                                  # the host variant gives the same matrix
        got_M, got_inv = one.read()
        assert np.array_equal(got_M, M) and np.array_equal(got_inv, inv), (n, "host")
        one.close()
    got_M, got_inv = conf.read()                                # accumulated across calls
    assert np.array_equal(got_M, acc_M) and np.array_equal(got_inv, acc_inv)
    conf.reset()
    assert not conf.read()[0].any() and not conf.read()[1].any()
    conf.close()


@pytest.mark.parametrize("K", [21, 255])
def test_all_pixels_in_one_bin(torch_cuda, K):
    torch = torch_cuda
    n = 6_000_001
    conf = api.Confusion(K)
    gt = torch.full((n,), K - 1, dtype=torch.uint8, device="cuda")
    pred = torch.full((n,), K - 1, dtype=torch.int32, device="cuda")
    conf.add_dev(gt, pred)
    conf.add_dev(gt[1:], pred[1:].to(torch.uint8))
    M, inv = conf.read()
    assert M[K - 1, K - 1] == 2 * n - 1 and M.sum() == 2 * n - 1 and not inv.any()
    conf.close()


def test_host_variant_streams_many_chunks(torch_cuda):
    """More pixels than the staging holds (4 Mi per chunk): the chunks alternate between the two slots."""
    rng = np.random.RandomState(3)
    gt, pred = labels(rng, 19_000_003, 21, np.int32)
    conf = api.Confusion(21)
    conf.add_host(gt, pred)
    conf.add_host(gt[5:], pred[5:].astype(np.int64))            # int64 is narrowed on the host
    M1, inv1 = want_matrix(gt, pred, 21)
    M2, inv2 = want_matrix(gt[5:], pred[5:], 21)
    M, inv = conf.read()
    assert np.array_equal(M, M1 + M2) and np.array_equal(inv, inv1 + inv2)
    conf.close()


def test_bad_arguments(torch_cuda):
    torch = torch_cuda
    with pytest.raises(api.DsrgError):
        api.Confusion(0)
    with pytest.raises(api.DsrgError):
        api.Confusion(256)
    conf = api.Confusion(21)
    g = torch.zeros(8, dtype=torch.uint8, device="cuda")
    with pytest.raises(TypeError):
        conf.add_dev(g, torch.zeros(8, dtype=torch.int64, device="cuda"))
    with pytest.raises(ValueError):
        conf.add_dev(g, torch.zeros(9, dtype=torch.uint8, device="cuda"))
    import ctypes as C
    L = conf._L
    assert L.dsrg_confusion_add_dev(conf.h, 4, C.c_void_p(g.data_ptr()), C.c_void_p(g.data_ptr() + 1), 4, None) != 0
    assert L.dsrg_confusion_add_dev(conf.h, 4, C.c_void_p(g.data_ptr()), C.c_void_p(g.data_ptr()), 2, None) != 0
    conf.close()


@pytest.mark.parametrize("K", [2, 21, 22, 81, 82])
def test_dropin_classes_match_frozen_reference(torch_cuda, K):
    g = load_golden("eval_ref.npz")
    items = [(g["gt_%d_%d" % (K, i)].flatten(), g["pred_%d_%d" % (K, i)].flatten()) for i in range(3)]
    ev, ap, ev_add = metrics.ConfusionMatrix(K), metrics.APConfusionMatrix(K), metrics.ConfusionMatrix(K)
    ev.addM(ev.generateM_all(items))
    for it in items:
        ap.addM(ap.generateM(it))
        gt, pred = it
        bad = gt >= K
        ev_add.add(np.where(bad, 255, gt).astype(np.uint8), np.where(bad, 0, pred))
    assert np.array_equal(ev.M, g["M_%d" % K]) and np.array_equal(ap.M, g["M_%d" % K])
    assert np.array_equal(ev_add.M, g["M_add_%d" % K])
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        r, a, (j, per, _) = ev.recall(), ev.accuracy(), ev.jaccard()
        (ar, arp), (aa, aap), (aj, ajp, _) = ap.recall(), ap.accuracy(), ap.jaccard()

    def same(x, y):
        x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
        return bool(np.all((x == y) | (np.isnan(x) & np.isnan(y))))
    assert same(r, g["ev_recall_%d" % K]) and same(a, g["ev_accuracy_%d" % K])
    assert same(j, g["ev_jaccard_%d" % K]) and same(per, g["ev_jaccard_per_%d" % K])
    assert same(ar, g["ap_recall_%d" % K]) and same(arp, g["ap_recall_per_%d" % K])
    assert same(aa, g["ap_accuracy_%d" % K]) and same(aap, g["ap_accuracy_per_%d" % K])
    assert same(aj, g["ap_jaccard_%d" % K]) and same(ajp, g["ap_jaccard_per_%d" % K])
    # get_confusion_matrix: the intended matrix; the reference's differs wherever its uint8 gt * K wrapped
    for i, (gt, pred) in enumerate(items):
        keep = gt != 255
        got = metrics.get_confusion_matrix(gt[keep], pred[keep].astype(np.int64), K)
        assert np.array_equal(got, want_matrix(gt[keep], pred[keep], K)[0].astype(np.float64))
        if K in (21, 22, 81, 82):
            assert not np.array_equal(got, g["coco_%d_%d" % (K, i)])
    with pytest.raises(IndexError):
        ev.generateM((np.array([1], np.uint8), np.array([K])))


def test_get_confusion_matrix_does_not_wrap(torch_cuda):
    g = load_golden("eval_ref.npz")
    got = metrics.get_confusion_matrix(g["wrap_gt"], g["wrap_pred"], 81)
    assert got[4, 4] == 2 and got[0, 72] == 0 and g["wrap_ref"][0, 72] == 2
    mean, iu = metrics.mean_iu(got)
    assert iu[4] == 1.0


def labels_agree(got, want_labels, want_probs, sel=None, margin=4 * TOL):
    """tests/test_gpu_post.py's rule: label maps equal except where the oracle's top-2 margin is a near-tie."""
    bad = got != want_labels
    if not bad.any():
        return 0
    p = want_probs if sel is None else want_probs[:, :, sel]
    top2 = np.sort(p, axis=2)[:, :, -2:]
    gap = top2[:, :, 1] - top2[:, :, 0]
    assert (gap[bad] <= margin).all(), "label differs where the oracle's margin is %g" % gap[bad].max()
    return int(bad.sum())


@pytest.mark.parametrize("H,W,sizes,index", [(90, 120, (31, 41), 0), (75, 64, (41,), 1)])
def test_predict_mask_ms_81_labels(torch_cuda, H, W, sizes, index):
    s = synth.make_score_blobs(200 + index, H, W, sizes, C=81)
    for smooth in (True, False):
        want_lab, want_p = post_oracle.predict_mask_ms(s["image"], s["blobs"], smooth=smooth)
        got_lab, got_p = postprocess.predict_mask_ms(s["image"], s["blobs"], smooth=smooth, return_probs=True)
        assert got_p.shape == (H, W, 81)
        if smooth:
            assert np.abs(got_p - want_p).max() <= TOL
            assert labels_agree(got_lab, want_lab, want_p) <= 1e-3 * H * W
            assert len(np.unique(want_lab)) >= 2
        else:
            np.testing.assert_allclose(got_p, want_p, rtol=2e-6, atol=1e-9)
            labels_agree(got_lab, want_lab, want_p, margin=1e-6)


@pytest.mark.parametrize("all_ids", [False, True], ids=["tags", "81ids"])
def test_predict_mask_gt_81_labels(torch_cuda, all_ids):
    H, W = 80, 100
    s = synth.make_score_blobs(210 + all_ids, H, W, (41,), C=81)
    tags = np.arange(1, 81) if all_ids else s["tags"]
    sel = [0] + list(tags)
    assert len(sel) == (81 if all_ids else len(sel))
    for smooth in (True, False):
        want_lab, want_p = post_oracle.predict_mask_gt(s["image"], s["blobs"][0], tags, smooth=smooth)
        got_lab, got_p = postprocess.predict_mask_gt(s["image"], s["blobs"][0], tags, smooth=smooth,
                                                     return_probs=True)
        assert set(np.unique(got_lab)) <= set(sel)
        if smooth:
            assert np.abs(got_p - want_p).max() <= TOL
            labels_agree(got_lab, want_lab, want_p, sel)
        else:
            np.testing.assert_allclose(got_p, want_p, rtol=4e-6, atol=1e-9)
            labels_agree(got_lab, want_lab, want_p, sel, margin=1e-6)


def test_coco_loop_predict_then_score_on_one_stream(torch_cuda):
    """test-coco.py's loop on the device: predict_mask_dev, then Confusion.add_dev of the same label map on the
    same stream, image sizes changing, the engine's CUDA graphs on (the sizes repeat, so passes are replayed)."""
    torch = torch_cuda
    K = 81
    rng = np.random.RandomState(11)
    sizes = [(90, 120), (120, 90), (64, 80)]
    eng = pool.engine_for(120, 120, K)
    eng.set_graphs(True)
    r0 = eng.graph_replays
    stream = torch.cuda.Stream()
    conf = api.Confusion(K)
    want = np.zeros((K, K), np.uint64)
    bufs = {}
    with torch.cuda.stream(stream):
        for rnd in range(3):
            for i, (H, W) in enumerate(sizes):
                if (H, W) not in bufs:   # per size the same buffers, so the engine replays its graph for them
                    s = synth.make_score_blobs(300 + i, H, W, (41,), C=K)
                    bufs[H, W] = ([torch.from_numpy(b).cuda() for b in s["blobs"]], torch.from_numpy(s["image"]).cuda(),
                                  torch.empty((H, W), dtype=torch.int32, device="cuda"))
                blobs, im, res = bufs[H, W]
                eng = pool.engine_for(H, W, K)
                eng.predict_mask_dev(blobs, im, res, stream=stream.cuda_stream)
                gt = rng.randint(0, K, (H, W)).astype(np.uint8)
                gt[:5] = 255
                conf.add_dev(torch.from_numpy(gt).cuda(), res, stream=stream.cuda_stream)
                want += want_matrix(gt, res.cpu().numpy(), K)[0]
    M, inv = conf.read()
    assert np.array_equal(M, want) and not inv.any()
    assert eng.graph_replays - r0 >= 3
    conf.close()
