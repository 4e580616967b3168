"""GPU tests of ImageSegDataLayer (pylayers/pylayers/layer.py), the stage-2 training input:
dsrg_seg_data_forward_{host,dev} against the numpy restatement (oracle/seg_data_oracle.py), and the drop-in layer and
SimpleTransformer against the frozen outputs of the reference's own classes (tests/golden/seg_data_ref.npz)."""
import ctypes as C
import importlib.util
import os
import random

import numpy as np
import pytest

import fake_caffe
from conftest import GOLDEN, load_golden

fake_caffe.install()
from dsrg_b200 import _lib, api, synth  # noqa: E402
from oracle import seg_data_oracle as oracle  # noqa: E402
from pylayers import layer as seg_layer  # noqa: E402
from pylayers import pylayers as _pl  # noqa: E402
from test_seg_data_cpu import matches_golden  # noqa: E402

pytestmark = pytest.mark.gpu

_spec = importlib.util.spec_from_file_location("make_seg_data_golden", os.path.join(GOLDEN, "make_seg_data_golden.py"))
make_golden = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(make_golden)
MEAN = make_golden.MEAN
VOC_MEAN = (104.0, 117.0, 123.0)


def restated(images, labels, h_off, w_off, flips, crop, mean, scale, swap=False, ignore=255):
    """The restatement with the windows and flips given -> (images (B,3,h,w), labels (B,1,h,w) or None)."""
    crop_h, crop_w = crop
    ims, labs = [], []
    for b, image in enumerate(images):
        if labels is None:
            pad_h, pad_w = max(crop_h - image.shape[0], 0), max(crop_w - image.shape[1], 0)
            im = oracle.pad_bottom_right(oracle.normalised(image, mean, scale, swap), pad_h, pad_w, 0.0)
            im = oracle.crop_chw(im, h_off[b], w_off[b], crop_h, crop_w)
            ims.append(im[:, :, ::-1] if flips and flips[b] else im)
        else:
            im, lab = oracle.transform(image, labels[b], crop, mean, scale, h_off[b], w_off[b],
                                       flips[b] if flips else 0, ignore)
            ims.append(im)
            labs.append(lab[None])
    return np.stack(ims), (np.stack(labs) if labels is not None else None)


def make_batch(sizes, label_sizes, crop, seed, phase="Train"):
    """Noise images, label maps with the background, two classes and ignore pixels, and windows drawn like the
    reference's (seeded), alternating flips."""
    rng = np.random.RandomState(seed)
    random.seed(seed)
    images = [synth.make_image(np.random.RandomState(seed * 100 + i), H, W, "noise") for i, (H, W) in enumerate(sizes)]
    labels = []
    for i, (H, W) in enumerate(label_sizes or sizes):
        values = np.array([0, rng.randint(1, 21), rng.randint(1, 21), 255], np.uint8)
        labels.append(values[rng.randint(0, 4, (H, W))])
    offs = [oracle.draw(lab.shape, crop, phase)[:2] for lab in labels]
    return images, labels, [o[0] for o in offs], [o[1] for o in offs], [i % 2 for i in range(len(sizes))]


def check_both(torch, eng, images, labels, h_off, w_off, flips, crop, mean, scale, swap=False, ignore=255):
    want = restated(images, labels, h_off, w_off, flips, crop, mean, scale, swap, ignore)
    pad = oracle.pad_byte(ignore)
    got = eng.seg_data_forward_host(images, labels, h_off, w_off, crop, mean, scale, flips, swap, pad)
    assert np.array_equal(got[0], want[0])
    assert (got[1] is None) == (labels is None)
    if labels is not None:
        assert np.array_equal(got[1], want[1])
    B = len(images)
    d_out = (torch.full((B, 3) + tuple(crop), 7.0, device="cuda"),
             None if labels is None else torch.full((B, 1) + tuple(crop), 7.0, device="cuda"))
    eng.seg_data_forward_dev([torch.from_numpy(im).cuda() for im in images],
                             None if labels is None else [torch.from_numpy(lab).cuda() for lab in labels],
                             h_off, w_off, d_out[0], d_out[1], mean, scale, flips, swap, pad)
    torch.cuda.synchronize()
    assert np.array_equal(d_out[0].cpu().numpy(), want[0])
    if labels is not None:
        assert np.array_equal(d_out[1].cpu().numpy(), want[1])
    return want


CONFIGS = [   # (name, image sizes, label sizes (None: the image's), crop, mean, scale, ignore_label, phase)
    ("voc", [(375, 500), (500, 375), (333, 500), (281, 500)], None, (321, 321), VOC_MEAN, 1.0, 255, "Train"),
    ("voc_test", [(375, 500), (500, 375), (366, 321), (321, 366)], None, (321, 321), MEAN, 1.0, 255, "Test"),
    ("voc_scale", [(375, 500), (500, 375)], None, (321, 321), [128, 128, 128], 0.017, 300, "Train"),
    ("img_larger", [(380, 510), (330, 340)], [(375, 500), (300, 300)], (321, 321), VOC_MEAN, 1.0, 254.5, "Train"),
    ("thin", [(1, 9), (13, 1), (1, 1)], None, (3, 5), MEAN, 1.0, -5, "Train"),
    ("batch20", [(7 + i, 30 - i) for i in range(20)], None, (15, 17), MEAN, 1.0, 255, "Train"),
]


@pytest.mark.parametrize("cfg", CONFIGS, ids=[c[0] for c in CONFIGS])
def test_entry_points_match_restatement(torch_cuda, cfg):
    name, sizes, label_sizes, crop, mean, scale, ignore, phase = cfg
    images, labels, h_off, w_off, flips = make_batch(sizes, label_sizes, crop, seed=len(name), phase=phase)
    eng = api.Engine(len(images), 1, 1, 1)
    want = check_both(torch_cuda, eng, images, labels, h_off, w_off, flips, crop, mean, scale, ignore=ignore)
    assert (want[1] == oracle.pad_byte(ignore)).any() or all(
        lab.shape[0] >= crop[0] and lab.shape[1] >= crop[1] for lab in labels)
    # the image-only paths on the same images: preprocess(image) and pre_test_image, centred windows
    centre = [(oracle.centred(max(im.shape[0], crop[0]), crop[0]), oracle.centred(max(im.shape[1], crop[1]), crop[1]))
              for im in images]
    for swap in (False, True):
        check_both(torch_cuda, eng, images, None, [c[0] for c in centre], [c[1] for c in centre], None, crop, mean,
                   scale, swap)
    eng.close()


@pytest.mark.parametrize("case", make_golden.CASES, ids=[c[0] for c in make_golden.CASES])
def test_entry_points_on_the_golden_cases(torch_cuda, case):
    """Each frozen case's images, windows and flips through both entry points against the restatement."""
    name, kind, sizes, label_sizes, B, params, seed = case
    p = oracle.params_of(params)
    files, indexlist, root = make_golden.case_files(case)
    images = [files[root + im] for im, _ in indexlist]
    if kind == "layer":
        labels = [files[root + lab] for _, lab in indexlist]
        random.seed(seed)
        np.random.seed(seed)
        draws = [oracle.draw(lab.shape, p["crop_size"], p["phase"], p["mirror"]) for lab in labels]
        h_off, w_off, flips = ([d[k] for d in draws] for k in range(3))
    else:
        labels, flips = None, None
        crop = p["crop_size"]
        h_off = [oracle.centred(max(im.shape[0], crop[0]), crop[0]) for im in images]
        w_off = [oracle.centred(max(im.shape[1], crop[1]), crop[1]) for im in images]
    eng = api.Engine(len(images), 1, 1, 1)
    check_both(torch_cuda, eng, images, labels, h_off, w_off, flips, p["crop_size"], p["mean"], p["scale"],
               kind == "pre_test", p["ignore_label"])
    eng.close()


def _write_list(tmp_path, indexlist):
    src = tmp_path / "train.txt"
    src.write_text("".join("%s %s\n" % tuple(e) for e in indexlist))
    return str(src)


def _layer(tmp_path, indexlist, root, B, params):
    layer = seg_layer.ImageSegDataLayer()
    layer.param_str = repr(dict(params, batch_size=B, root_folder=root, source=_write_list(tmp_path, indexlist)))
    top = [fake_caffe.Blob() for _ in range(2)]
    layer.setup([], top)
    layer.reshape([], top)
    return layer, top


def _same_states(states):
    assert random.getstate() == states[0]
    assert all(np.array_equal(a, b) for a, b in zip(np.random.get_state(), states[1]))


@pytest.mark.parametrize("case", make_golden.CASES, ids=[c[0] for c in make_golden.CASES])
def test_layer_matches_frozen_reference(torch_cuda, tmp_path, monkeypatch, case):
    """The drop-in, reading the in-memory files through _imread, equals the reference's own classes, and leaves both
    random states where the restatement leaves them."""
    name, kind, sizes, label_sizes, B, params, seed = case
    files, indexlist, root = make_golden.case_files(case)
    original = [list(e) for e in indexlist]
    monkeypatch.setattr(_pl, "_imread", lambda path, flag: files[path])
    g = load_golden("seg_data_ref.npz")
    if kind == "layer":
        layer, top = _layer(tmp_path, indexlist, root, B, params)
        random.seed(seed)
        np.random.seed(seed)
        layer.forward([], top)
        loader = layer.batch_loader
        matches_golden(g, name, top[0].data, top[1].data, loader._cur, make_golden.order_of(loader.indexlist,
                                                                                             original))
        states = random.getstate(), np.random.get_state()
        random.seed(seed)
        np.random.seed(seed)
        oracle.seg_data_forward(lambda p_, f: files[p_], [list(e) for e in original], 0, root, B, params)
        _same_states(states)
    else:
        t = seg_layer.SimpleTransformer(dict(params))
        fn = t.preprocess if kind == "preprocess" else t.pre_test_image
        matches_golden(g, name, np.stack([fn(files[root + im]) for im, _ in indexlist]))


def test_batch_loader_and_preprocess_are_single_image_calls(torch_cuda, tmp_path, monkeypatch):
    case = make_golden.CASES[0]
    files, indexlist, root = make_golden.case_files(case)
    monkeypatch.setattr(_pl, "_imread", lambda path, flag: files[path])
    params = dict(case[5], batch_size=1, root_folder=root, source=_write_list(tmp_path, indexlist))
    loader = seg_layer.BatchLoader(dict(params))
    random.seed(3)
    np.random.seed(3)
    got = [loader.load_next_image() for _ in range(2)]
    random.seed(3)
    np.random.seed(3)
    want = [oracle.preprocess(files[root + im], files[root + lab], params) for im, lab in indexlist]
    for (gi, gl), (wi, wl) in zip(got, want):
        assert gi.shape == wi.shape and gl.shape == wl.shape
        assert np.array_equal(gi, wi) and np.array_equal(gl, wl)
    assert loader._cur == 2
    t = loader.transformer
    im, lab = files[root + indexlist[0][0]], files[root + indexlist[0][1]]
    random.seed(4)
    np.random.seed(4)
    got = t.preprocess(im, lab)
    random.seed(4)
    np.random.seed(4)
    want = oracle.preprocess(im, lab, params)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])


def test_bad_arguments_are_refused_before_any_launch(torch_cuda):
    torch = torch_cuda
    dev = torch.cuda.current_device()
    L = _lib.lib()
    eng = api.Engine(2, 1, 1, 1)
    images, labels, _, _, _ = make_batch([(6, 7), (5, 4)], None, (4, 4), seed=9)
    d_im = [torch.from_numpy(im).cuda() for im in images]
    d_lab = [torch.from_numpy(lab).cuda() for lab in labels]
    d_out = [torch.zeros(2, 3, 4, 4, device="cuda"), torch.zeros(2, 1, 4, 4, device="cuda")]
    h_out = [np.zeros((2, 3, 4, 4), np.float32), np.zeros((2, 1, 4, 4), np.float32)]
    mean = np.array(MEAN)

    def args(dev_side, B=2, Hs=(6, 5), Ws=(7, 4), Hl=(6, 5), Wl=(7, 4), ho=(1, 0), wo=(2, 0), crop=(4, 4), pad=255,
             ptrs=None):
        p = ptrs or ([t.data_ptr() for t in d_im] if dev_side else [im.ctypes.data for im in images])
        lp = [t.data_ptr() for t in d_lab] if dev_side else [lab.ctypes.data for lab in labels]
        ints = lambda v: (C.c_int * 2)(*v)  # noqa: E731
        a = [eng.h, (C.c_void_p * 2)(*p), ints(Hs), ints(Ws), (C.c_void_p * 2)(*lp), ints(Hl), ints(Wl), B, ints(ho),
             ints(wo), None, crop[0], crop[1], C.c_void_p(mean.ctypes.data), 1.0, 0, pad]
        a += [C.c_void_p(o.data_ptr()) for o in d_out] if dev_side else [C.c_void_p(o.ctypes.data) for o in h_out]
        return a + [None] if dev_side else a

    calls = [(L.dsrg_seg_data_forward_dev, True), (L.dsrg_seg_data_forward_host, False)]
    eng.take_launch_count()
    for fn, dev_side in calls:
        assert fn(*args(dev_side)) == _lib.OK
    assert eng.take_launch_count() == 2
    torch.cuda.synchronize()
    for fn, dev_side in calls:
        for k in (1, 2, 3, 5, 6, 8, 9, 13, 17, 18):   # required pointers (Hl, Wl and labels_out: with labels)
            a = args(dev_side)
            a[k] = None
            assert fn(*a) == _lib.E_INVALID, (fn, k)
        for bad in (dict(B=0), dict(B=3), dict(Hs=(0, 5)), dict(Ws=(7, -1)), dict(Hl=(6, 0)), dict(crop=(0, 4)),
                    dict(crop=(4, 0)), dict(pad=-1), dict(pad=256), dict(ho=(-1, 0)), dict(wo=(0, -2)),
                    dict(ho=(3, 0)),                   # leaves the label (6 rows, window of 4 from row 3)
                    dict(Hs=(6, 3)),                   # leaves the image: 3 rows, no padding (the label has 5)
                    dict(Ws=(7, 3), Wl=(7, 3), wo=(2, 1)),   # padded to 4 columns, the window starts at 1
                    dict(ptrs=[None, 1] if not dev_side else [d_im[0].data_ptr(), None])):
            assert fn(*args(dev_side, **bad)) == _lib.E_INVALID, (fn, bad)
        assert eng.take_launch_count() == 0
        assert torch.cuda.current_device() == dev
    # image only: the label arrays, their sizes and labels_out are not read
    for fn, dev_side in calls:
        a = args(dev_side, ho=(1, 0), wo=(1, 0))
        a[4] = a[5] = a[6] = None
        a[18] = None
        assert fn(*a) == _lib.OK
        a = args(dev_side, ho=(3, 0), wo=(1, 0))   # padding from the image now: 6 rows, a window of 4 from row 3
        a[4] = None
        assert fn(*a) == _lib.E_INVALID
    assert eng.take_launch_count() == 2
    torch.cuda.synchronize()
    eng.close()


def test_layer_window_that_does_not_fit(torch_cuda, tmp_path, monkeypatch):
    """An image shorter than its label: numpy's broadcast ValueError, after the draws of that image, before any
    device call."""
    files = {"/d/a.jpg": np.zeros((300, 400, 3), np.uint8), "/d/a.png": np.zeros((300, 400), np.uint8),
             "/d/b.jpg": np.zeros((200, 400, 3), np.uint8), "/d/b.png": np.zeros((400, 400), np.uint8)}
    indexlist = [["a.jpg", "a.png"], ["b.jpg", "b.png"]]
    monkeypatch.setattr(_pl, "_imread", lambda path, flag: files[path])
    params = {"crop_size": (321, 321), "mirror": True}
    layer, top = _layer(tmp_path, indexlist, "/d/", 2, params)
    eng = _pl._engine(2, 1, 1, 1)
    random.seed(8)
    np.random.seed(8)
    eng.take_launch_count()
    with pytest.raises(ValueError) as got:
        layer.forward([], top)
    assert eng.take_launch_count() == 0
    states = random.getstate(), np.random.get_state()
    random.seed(8)
    np.random.seed(8)
    with pytest.raises(ValueError) as want:
        oracle.seg_data_forward(lambda p, f: files[p], [list(e) for e in indexlist], 0, "/d/", 2, params)
    assert str(got.value) == str(want.value) and "could not broadcast input array from shape (3," in str(got.value)
    _same_states(states)
    assert layer.batch_loader._cur == 2


def test_layer_errors_name_the_missing_file(torch_cuda, tmp_path, monkeypatch):
    layer, top = _layer(tmp_path, [["a.jpg", "a.png"]], "/d/", 1, {"crop_size": (5, 5)})
    monkeypatch.setattr(_pl, "_imread", lambda path, flag: None)   # what cv2.imread returns for a missing file
    with pytest.raises(IOError, match="/d/a.jpg"):
        layer.forward([], top)


def test_layer_engine_is_small_and_tops_are_written_in_place(torch_cuda, tmp_path, monkeypatch):
    """train-f.prototxt's shape: batch 10, crop 321, VOC-sized images.  The layer's engine stays far below a
    CRF-sized one."""
    files, lines = {}, []
    for i in range(12):
        H, W = (375, 500) if i % 2 else (500, 375)
        files["/d/%d.jpg" % i] = synth.make_image(np.random.RandomState(i), H, W, "noise")
        files["/d/%d.png" % i] = np.random.RandomState(50 + i).randint(0, 21, (H, W)).astype(np.uint8)
        lines.append(["%d.jpg" % i, "%d.png" % i])
    monkeypatch.setattr(_pl, "_imread", lambda path, flag: files[path])
    layer, top = _layer(tmp_path, lines, "/d/", 10, {"mean": VOC_MEAN, "mirror": True, "crop_size": (321, 321)})
    bufs = [t.data for t in top]
    random.seed(1)
    np.random.seed(1)
    layer.forward([], top)
    assert all(t.data is b for t, b in zip(top, bufs))
    random.seed(1)
    np.random.seed(1)
    want = oracle.seg_data_forward(lambda p, f: files[p], [list(e) for e in lines], 0, "/d/", 10,
                                   {"mean": VOC_MEAN, "mirror": True, "crop_size": (321, 321)})
    assert np.array_equal(top[0].data, want[0]) and np.array_equal(top[1].data, want[1])
    small = _pl._engine(10, 1, 1, 1).device_bytes
    big = api.Engine(10, 321, 321, 21)
    assert 0 < small < big.device_bytes / 10, (small, big.device_bytes)
    big.close()


def test_layer_reads_png_files_with_cv2(torch_cuda, tmp_path):
    cv2 = pytest.importorskip("cv2")
    case = ("png", "layer", [(37, 45), (50, 31)], None, 3, {"crop_size": (41, 41), "mean": MEAN, "mirror": True}, 6)
    files, indexlist, _ = make_golden.case_files(case)
    root = str(tmp_path) + "/"
    os.makedirs(root + "JPEGImages")
    os.makedirs(root + "SegmentationClassAug")
    for path, a in files.items():
        assert cv2.imwrite(root + path[len(make_golden.DATA_ROOT):].replace(".jpg", ".png"), a)
    indexlist = [[im.replace(".jpg", ".png"), lab] for im, lab in indexlist]
    layer, top = _layer(tmp_path, indexlist, root, 3, case[5])
    random.seed(6)
    np.random.seed(6)
    layer.forward([], top)
    random.seed(6)
    np.random.seed(6)
    want = oracle.seg_data_forward(cv2.imread, [list(e) for e in indexlist], 0, root, 3, case[5])
    assert np.array_equal(top[0].data, want[0]) and np.array_equal(top[1].data, want[1])
