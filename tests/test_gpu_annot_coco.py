"""GPU tests of AnnotationLayerCOCO (pylayers.py:389-512): dsrg_annotation_coco_forward_{host,dev} against the numpy
restatement (oracle/annot_coco_oracle.py) and the frozen outputs of the reference's own class
(tests/golden/annot_coco_ref.npz), the drop-in layer, and one 81-label training step through the drop-in classes."""
import ctypes as C
import importlib.util
import os

import numpy as np
import pytest

import fake_caffe
from conftest import GOLDEN, load_golden

fake_caffe.install()
import pylayers  # noqa: E402
from dsrg_b200 import _lib, api, synth  # noqa: E402
from oracle import annot_coco_oracle, crf_oracle, loss_oracle, srg_oracle  # noqa: E402
from pylayers import pylayers as _pl  # noqa: E402
from test_annot_coco_cpu import matches_golden  # noqa: E402

pytestmark = pytest.mark.gpu

_spec = importlib.util.spec_from_file_location("make_annot_coco_golden",
                                               os.path.join(GOLDEN, "make_annot_coco_golden.py"))
make_golden = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(make_golden)
MEAN = make_golden.MEAN


def batch(sizes, new_size, seed, ignore=255, flip_every=2):
    """Noise images of the given sizes, label maps at the cue size with two classes, the background and ignore
    pixels, and alternating mirror flags."""
    rng = np.random.RandomState(seed)
    h, w = new_size[0] // 8 + 1, new_size[1] // 8 + 1
    images = [synth.make_image(np.random.RandomState(seed * 100 + i), H, W, "noise") for i, (H, W) in enumerate(sizes)]
    labels = np.empty((len(sizes), h, w), np.uint8)
    for i in range(len(sizes)):
        values = np.array([0] + list(rng.choice(np.arange(1, 81), 2, replace=False)) + [ignore])
        labels[i] = values[rng.randint(0, 4, (h, w))]
    flips = [int(i % flip_every == 1) for i in range(len(sizes))]
    return images, labels, flips


def restated(images, labels, flips, new_size, ignore=255):
    outs = [annot_coco_oracle.coco_preprocess(im, lab, new_size, MEAN, -1 if f else 1, ignore)
            for im, lab, f in zip(images, labels, flips)]
    return tuple(np.stack([o[k] for o in outs]).astype(np.float32) for k in (2, 1, 0))


CONFIGS = [   # (name, image sizes, new_size, ignore_label)
    ("voc", [(375, 500), (500, 375), (333, 500)], (321, 321), 255),
    ("coco", [(480, 640), (640, 480), (427, 640), (612, 612)], (321, 321), 255),
    ("thin_up", [(1, 9), (13, 1), (1, 1), (4, 5)], (17, 23), 255),     # H or W of 1, upsampling
    ("cval", [(40, 51), (51, 40)], (45, 45), 3),                       # 51 -> 45: scipy's 0 column
    ("batch20", [(7 + i, 30 - i) for i in range(20)], (25, 31), 255),  # more images than DSRG_PREP_MAX_SCALES
]


@pytest.mark.parametrize("cfg", CONFIGS, ids=[c[0] for c in CONFIGS])
def test_entry_points_match_restatement(torch_cuda, cfg):
    torch = torch_cuda
    name, sizes, new_size, ignore = cfg
    images, labels, flips = batch(sizes, new_size, seed=len(name), ignore=ignore)
    B, h, w = labels.shape
    eng = api.Engine(B, h, w, 81)
    want = restated(images, labels, flips, new_size, ignore)
    got = eng.annotation_coco_forward_host(images, labels, new_size, MEAN, flips, ignore)
    for g, wnt in zip(got, want):
        assert g.shape == wnt.shape and np.array_equal(g, wnt), name
    assert want[1].sum() > 0 and want[0].sum() > 0
    d_images = [torch.from_numpy(im).cuda() for im in images]
    outs = (torch.full((B, 1, 1, 81), 7.0, device="cuda"), torch.full((B, 81, h, w), 7.0, device="cuda"),
            torch.full((B, 3) + tuple(new_size), 7.0, device="cuda"))
    bad = torch.zeros(B, dtype=torch.int32, device="cuda")
    eng.annotation_coco_forward_dev(d_images, torch.from_numpy(labels).cuda(), *outs, MEAN, flips, ignore, bad)
    torch.cuda.synchronize()
    for d, g in zip(outs, got):
        assert np.array_equal(d.cpu().numpy(), g), name
    assert (bad.cpu().numpy() == -1).all()
    eng.close()


def test_out_of_range_labels(torch_cuda):
    """_host refuses them with numpy's message before any launch; _dev skips them and reports the first pixel."""
    torch = torch_cuda
    images, labels, flips = batch([(30, 40), (20, 10), (9, 9)], (17, 17), seed=5)
    eng = api.Engine(3, 3, 3, 81)
    labels[1, 0, 2] = 90
    labels[1, 2, 1] = 200
    labels[2, 1, 1] = 81
    eng.take_launch_count()
    with pytest.raises(api.DsrgError, match="index 90 is out of bounds for axis 0 with size 81"):
        eng.annotation_coco_forward_host(images, labels, (17, 17), MEAN, flips)
    assert eng.take_launch_count() == 0
    outs = (torch.zeros(3, 1, 1, 81, device="cuda"), torch.zeros(3, 81, 3, 3, device="cuda"),
            torch.zeros(3, 3, 17, 17, device="cuda"))
    bad = torch.zeros(3, dtype=torch.int32, device="cuda")
    eng.annotation_coco_forward_dev([torch.from_numpy(im).cuda() for im in images], torch.from_numpy(labels).cuda(),
                                    *outs, MEAN, flips, 255, bad)
    torch.cuda.synchronize()
    assert bad.cpu().numpy().tolist() == [-1, 2, 4]
    clean = labels.copy()
    clean[clean >= 81] = 255   # what _dev writes: the out-of-range pixels count as ignored
    want = restated(images, clean, flips, (17, 17))
    for d, wnt in zip(outs, want):
        assert np.array_equal(d.cpu().numpy(), wnt)
    eng.close()


def test_bad_arguments_are_refused_before_any_launch(torch_cuda):
    torch = torch_cuda
    dev = torch.cuda.current_device()
    L = _lib.lib()
    eng = api.Engine(2, 3, 3, 81)
    images, labels, flips = batch([(6, 7), (5, 4)], (17, 17), seed=9)
    d_im = [torch.from_numpy(im).cuda() for im in images]
    d_lab = torch.from_numpy(labels).cuda()
    outs = [torch.zeros(2, 1, 1, 81, device="cuda"), torch.zeros(2, 81, 3, 3, device="cuda"),
            torch.zeros(2, 3, 17, 17, device="cuda")]
    mean = np.array(MEAN)
    h_out = [np.zeros(o.shape, np.float32) for o in outs]

    def args(dev_side, B=2, Hs=(6, 5), Ws=(7, 4), ptrs=None, new_h=17, new_w=17):
        p = ptrs or ([t.data_ptr() for t in d_im] if dev_side else [im.ctypes.data for im in images])
        a = [eng.h, (C.c_void_p * 2)(*p), (C.c_int * 2)(*Hs), (C.c_int * 2)(*Ws), B,
             C.c_void_p(d_lab.data_ptr() if dev_side else labels.ctypes.data), None, new_h, new_w,
             C.c_void_p(mean.ctypes.data), 255]
        a += [C.c_void_p(o.data_ptr()) for o in outs] if dev_side else [C.c_void_p(o.ctypes.data) for o in h_out]
        return a + [None, None] if dev_side else a

    calls = [(L.dsrg_annotation_coco_forward_dev, True), (L.dsrg_annotation_coco_forward_host, False)]
    eng.take_launch_count()
    for fn, dev_side in calls:
        assert fn(*args(dev_side)) == _lib.OK
    assert eng.take_launch_count() == 6
    torch.cuda.synchronize()
    for fn, dev_side in calls:
        required = [1, 2, 3, 5, 9, 11, 12, 13]
        for k in required:
            a = args(dev_side)
            a[k] = None
            assert fn(*a) == _lib.E_INVALID, (fn, k)
        for bad in (dict(B=0), dict(B=3), dict(Hs=(0, 5)), dict(Ws=(7, -1)), dict(new_h=0), dict(new_w=0),
                    dict(ptrs=[None, 1] if not dev_side else [d_im[0].data_ptr(), None])):
            assert fn(*args(dev_side, **bad)) == _lib.E_INVALID, (fn, bad)
        assert eng.take_launch_count() == 0
        assert torch.cuda.current_device() == dev
    eng.close()


def _write_list(tmp_path, indexlist):
    src = tmp_path / "list.txt"
    src.write_text("".join("%s %s\n" % tuple(e) for e in indexlist))
    return str(src)


def _params(src, root, case):
    name, sizes, shapes, B, new_size, mirror, ignore, seed = case
    return repr({"source": src, "root": root, "batch_size": B, "mean": MEAN, "new_size": new_size, "mirror": mirror,
                 "ignore_label": ignore})


@pytest.mark.parametrize("case", make_golden.CASES, ids=[c[0] for c in make_golden.CASES])
def test_layer_matches_frozen_reference(torch_cuda, tmp_path, monkeypatch, case):
    """The drop-in layer, reading the in-memory files through _imread, equals the reference's own forward."""
    files, indexlist, root = make_golden.case_files(case)
    original = [list(e) for e in indexlist]
    monkeypatch.setattr(_pl, "_imread", lambda path, flag: files[path])
    layer = pylayers.AnnotationLayerCOCO()
    layer.param_str = _params(_write_list(tmp_path, indexlist), root, case)
    top = [fake_caffe.Blob() for _ in range(3)]
    layer.setup([], top)
    layer.reshape([], top)
    np.random.seed(case[7])
    layer.forward([], top)
    matches_golden(load_golden("annot_coco_ref.npz"), case[0], top[0].data, top[1].data.astype(np.uint8),
                   top[2].data, layer._cur, make_golden.order_of(layer.indexlist, original))
    assert set(np.unique(top[1].data)) <= {0.0, 1.0}


def test_layer_errors(torch_cuda, tmp_path, monkeypatch):
    case = make_golden.CASES[0]
    files, indexlist, root = make_golden.case_files(case)
    src = _write_list(tmp_path, indexlist)
    layer = pylayers.AnnotationLayerCOCO()
    layer.param_str = _params(src, root, case)
    top = [fake_caffe.Blob() for _ in range(3)]
    layer.setup([], top)
    monkeypatch.setattr(_pl, "_imread", lambda path, flag: None)    # what cv2.imread returns for a missing file
    with pytest.raises(IOError, match=root + indexlist[0][0]):
        layer.forward([], top)
    bad = dict(files)
    lab = bad[root + indexlist[0][1]].copy()
    lab[0, 1] = 90
    bad[root + indexlist[0][1]] = lab
    monkeypatch.setattr(_pl, "_imread", lambda path, flag: bad[path])
    layer._cur = 0
    with pytest.raises(IndexError, match="^index 90 is out of bounds for axis 0 with size 81$"):
        layer.forward([], top)
    bad[root + indexlist[0][1]] = np.zeros((2, 3), np.uint8)          # neither (3, 3) nor broadcast to it
    layer._cur = 0
    with pytest.raises(ValueError):
        layer.forward([], top)


def test_layer_reads_png_files_with_cv2(torch_cuda, tmp_path):
    cv2 = pytest.importorskip("cv2")
    case = ("png", [(37, 45), (50, 31)], {}, 3, (33, 41), True, 255, 6)
    files, indexlist, _ = make_golden.case_files(case)
    root = str(tmp_path) + "/"
    os.makedirs(root + "JPEGImages")
    os.makedirs(root + "Annotations")
    for path, a in files.items():
        assert cv2.imwrite(root + path[len(make_golden.DATA_ROOT):].replace(".jpg", ".png"), a)
    indexlist = [[im.replace(".jpg", ".png"), lab] for im, lab in indexlist]
    want_list = [list(e) for e in indexlist]
    layer = pylayers.AnnotationLayerCOCO()
    layer.param_str = _params(_write_list(tmp_path, indexlist), root, case)
    top = [fake_caffe.Blob() for _ in range(3)]
    layer.setup([], top)
    np.random.seed(6)
    layer.forward([], top)
    np.random.seed(6)
    want = annot_coco_oracle.annotation_coco_forward(cv2.imread, want_list, 0, root, 3, MEAN, (33, 41), True)
    for t, wnt in zip(top, want[:3]):
        assert np.array_equal(t.data, wnt)
    assert layer._cur == want[3] and layer.indexlist == want_list


@pytest.mark.parametrize("share", ["1", "0"])
def test_81_label_training_step(torch_cuda, tmp_path, monkeypatch, share):
    """AnnotationLayerCOCO -> probs -> CRFLayer -> DSRGLayer -> BalancedSeedLossLayer and ConstrainLossLayer at 81
    labels, forward and backward, each top against its oracle.  The probs blob is the reference softmax of a seeded
    stand-in fc8 (the drop-in SoftmaxLayer stops at 32 labels)."""
    monkeypatch.setenv("DSRG_B200_SHARE_CRF", share)
    case = ("step", [(375, 500), (480, 640), (333, 500), (612, 612)], {}, 4, (321, 321), True, 255, 12)
    files, indexlist, root = make_golden.case_files(case)
    monkeypatch.setattr(_pl, "_imread", lambda path, flag: files[path])
    data = pylayers.AnnotationLayerCOCO()
    data.param_str = _params(_write_list(tmp_path, indexlist), root, case)
    d_top = [fake_caffe.Blob() for _ in range(3)]
    data.setup([], d_top)
    np.random.seed(12)
    data.forward([], d_top)
    labels, cues, images = (t.data for t in d_top)
    assert labels.shape == (4, 1, 1, 81) and cues.shape == (4, 81, 41, 41) and images.shape == (4, 3, 321, 321)
    rng = np.random.RandomState(12)
    fc8 = (rng.randn(4, 81, 41, 41) * 3).astype(np.float32)
    probs = loss_oracle.softmax_layer_forward(fc8).astype(np.float32)
    probs[0, 5, :4, :4] = 1e-6   # exercises the in-place clamp

    crf, b_crf, t_crf = fake_caffe.run_layer(pylayers.CRFLayer, [probs, images])
    clamped = np.maximum(probs, np.float32(1e-4))
    assert np.array_equal(b_crf[0].data, clamped)
    want_crf = crf_oracle.refinement(probs.copy(), images, 12.0)
    assert np.abs(np.exp(t_crf[0].data) - want_crf).max() <= 1e-4

    dsrg = pylayers.DSRGLayer()
    dsrg.param_str = "{'th1': 0.99, 'th2': 0.85}"
    bottom = [fake_caffe.Blob(labels), b_crf[0], fake_caffe.Blob(cues), b_crf[1]]
    s_top = [fake_caffe.Blob()]
    dsrg.setup(bottom, s_top)
    dsrg.reshape(bottom, s_top)
    dsrg.forward(bottom, s_top)
    seeds = s_top[0].data
    assert np.all(seeds >= cues)
    if share == "1":
        # one refinement serves both layers: the seeds are the reference SRG on its float64 renormalisation
        r64 = crf_oracle.renormalise(_pl._engine(4, 81, 41, 41).crf_last_marginals_host(4))
        assert np.abs(r64 - want_crf).max() <= 1e-4
        for b in range(4):
            assert np.array_equal(seeds[b], srg_oracle.srg_closed_form(labels[b, 0, 0], cues[b], r64[b], 0.99, 0.85))
    else:
        # the layer refines again, in pipelined chunks whose marginals are not all retained: against the CPU
        # refinement the seed maps may differ only where a marginal sits within 1e-4 of a threshold
        mism = sum(int((srg_oracle.srg_closed_form(labels[b, 0, 0], cues[b], want_crf[b], 0.99, 0.85)
                        != seeds[b]).sum()) for b in range(4))
        assert mism <= 1e-3 * seeds.size, mism
    s_top[0].diff[...] = 0.25
    dsrg.backward(s_top, [False, True, False, False], bottom)
    assert np.array_equal(bottom[1].diff, np.full(probs.shape, 0.25, np.float32))

    p = b_crf[0].data.copy()
    seed_loss, b_seed, t_seed = fake_caffe.run_layer(pylayers.BalancedSeedLossLayer, [p, seeds])
    want = loss_oracle.balanced_seed_loss(p, seeds)
    assert abs(float(t_seed[0].data[0]) - want) <= 1e-5 * abs(want)
    seed_loss.backward(t_seed, [True, False], b_seed)
    np.testing.assert_allclose(b_seed[0].diff, loss_oracle.balanced_seed_loss_grad(p, seeds), rtol=1e-5, atol=1e-9)

    logs = t_crf[0].data.copy()
    con, b_con, t_con = fake_caffe.run_layer(pylayers.ConstrainLossLayer, [p, logs])
    want = loss_oracle.constrain_loss(p, logs)
    assert abs(float(t_con[0].data[0]) - want) <= 2e-5 * abs(want)
    con.backward(t_con, [True, True], b_con)
    gp, gl = loss_oracle.constrain_loss_grad(p.astype(np.float64), logs.astype(np.float64))
    ratio = np.exp(logs.astype(np.float64)) / p
    safe = (np.abs(ratio - 0.05) > 1e-5) & (np.abs(ratio - 20) > 1e-3)
    np.testing.assert_allclose(b_con[0].diff[safe], gp[safe], rtol=2e-4, atol=1e-9)
    np.testing.assert_allclose(b_con[1].diff[safe], gl[safe], rtol=2e-4, atol=1e-9)

    # the CRF top's backward: (1 - result) * diff
    t_crf[0].diff[...] = 0.5
    crf.backward(t_crf, [True, False], b_crf)
    np.testing.assert_allclose(b_crf[0].diff, (1 - want_crf) * 0.5, atol=1e-4)
